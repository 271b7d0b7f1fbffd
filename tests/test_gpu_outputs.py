"""The output selection (rdn.set_outputs) on the GPU: wanted outputs bit-identical to the full window's on the eager and
the graphed path in both precisions, the stage launches a selection issues, streaming, the self-ensemble, the refusals,
and the test.py caller sequence with the three images it writes."""
from contextlib import contextmanager

import numpy as np
import pytest
import torch

from oracle import bin_oracle as O

pytestmark = pytest.mark.gpu
SELECTIONS = [(13, 8, 12), (13,), (9,), (0,), (4, 11)]
# backbone calls per stage (batch = calls x B) and ConvLSTM launches (the cells of one hand-off are one launch)
STAGE_CALLS = {None: [5, 6, 4, 2], (13, 8, 12): [4, 5, 3, 1], (13,): [4, 5, 3, 1], (9,): [4, 3, 2, 1], (0,): [1],
               (4, 11): [4, 2]}
LSTM_LAUNCHES = {None: 3, (13, 8, 12): 3, (13,): 3, (9,): 0, (0,): 0, (4, 11): 1}


def _new_net():
    from bin_b200 import rdn
    m = rdn.bin_stage4_lstm()
    m.load_state_dict(O.synth_state_dict(0), strict=True)
    return m.cuda().eval()


@pytest.fixture(scope="module")
def net():
    return _new_net()


@contextmanager
def selection(net, indices, unwanted="none", precision="fp16", ensemble=None):
    from bin_b200 import rdn
    rdn.set_outputs(net, indices, unwanted)
    rdn.set_precision(net, precision)
    rdn.set_self_ensemble(net, ensemble)
    try:
        yield net
    finally:
        rdn.set_outputs(net, None)
        rdn.set_precision(net, "fp16")
        rdn.set_self_ensemble(net, None)


def check_selected(got, full, wanted, unwanted="none"):
    assert isinstance(got, tuple) and len(got) == 14
    for i in range(14):
        if i in wanted:
            assert got[i].shape == full[i].shape and got[i].is_contiguous() and torch.equal(got[i], full[i]), i
        elif unwanted == "none":
            assert got[i] is None, i
        else:
            assert got[i].shape == full[i].shape and got[i].dtype == torch.float32 and got[i].device == full[i].device
            assert got[i].stride() == (0, 0, 0, 0) and not bool(got[i].any()), i
    assert len({got[i].data_ptr() for i in wanted}) == len(wanted)


@pytest.mark.parametrize("graph", ["0", "1"], ids=["eager", "graphed"])
@pytest.mark.parametrize("precision", ["fp16", "fp32"])
@pytest.mark.parametrize("B,H,W", [(1, 70, 98), (2, 70, 98), (1, 256, 256), (2, 256, 256)])
def test_wanted_outputs_are_bit_identical(net, monkeypatch, B, H, W, precision, graph):
    """Every selection against one full window, then back to the full window and to the first selection again: on the
    graphed path each switch must replace the captured graph."""
    monkeypatch.setenv("BIN_B200_GRAPH", graph)
    frames = [f.cuda() for f in O.synth_frames(6, B, H, W, seed=B * 1000 + H, smooth=True)]
    with torch.no_grad():
        with selection(net, None, precision=precision):
            full = net(*frames)
        assert all(o is not None for o in full)
        for k, wanted in enumerate(SELECTIONS + [None, SELECTIONS[0]]):
            unwanted = "zeros" if k % 2 else "none"
            with selection(net, wanted, unwanted, precision):
                got = net(*frames)
            check_selected(got, full, range(14) if wanted is None else wanted, unwanted)
    net.__dict__.pop("_graph_entry", None)


def _profiled_launches(fn):
    """(frame packer launches, ConvLSTM launches) of one fn() call.  The trace of a profiler that has run before in the
    process can lack the first kernels launched after it starts, so fn runs twice back to back with one elementwise
    kernel between the calls as a marker, and only what the trace holds after the marker is counted."""
    from torch.profiler import ProfilerActivity, profile
    fn()                                                    # warm-up: packed weights, workspace
    marker = torch.zeros(8, device="cuda")
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        marker.add_(1)
        fn()
        torch.cuda.synchronize()
    evs = sorted((ev for ev in prof.events() if ev.device_type == torch.autograd.DeviceType.CUDA),
                 key=lambda ev: ev.time_range.start)
    names = [ev.name for ev in evs]
    marks = [k for k, n in enumerate(names) if "elementwise_kernel" in n]
    assert len(marks) == 1, names[:4]
    names = names[marks[0] + 1:]
    return sum("::pack_frames_kernel" in n for n in names), sum("::convlstm_kernel" in n for n in names)


@pytest.mark.parametrize("wanted", [None] + SELECTIONS, ids=str)
def test_library_window_issues_one_packer_launch_per_live_stage(net, monkeypatch, wanted):
    """The module's window runs each stage that is left as one batched backbone launch, so the frame packer runs once per
    such stage, and the live cells of each recurrent hand-off as one ConvLSTM launch."""
    monkeypatch.setenv("BIN_B200_GRAPH", "0")
    frames = [f.cuda() for f in O.synth_frames(6, 1, 32, 48, seed=8)]
    with torch.no_grad(), selection(net, wanted):
        packs, lstms = _profiled_launches(lambda: net(*frames))
    assert (packs, lstms) == (len(STAGE_CALLS[wanted]), LSTM_LAUNCHES[wanted])


@pytest.mark.parametrize("B", [1, 2])
def test_streaming_follows_the_selection(net, monkeypatch, B):
    """9 frames, (13, 8, 12): each window equals the module's, the first costs 13 backbone calls (4 + 5 + 3 + 1: the pair
    of frames 0, 1 is never evaluated) and every later one 10 (1 + 5 + 3 + 1), in stage launches of those batch sizes."""
    from bin_b200 import rdn
    from bin_b200.streaming import StreamingBIN
    stages, real = [], rdn._launch_stage

    def counting(model, calls, outs, prec):
        stages.append((model.NFRAMES, len(calls), calls[0][0].shape[0]))
        return real(model, calls, outs, prec)

    monkeypatch.setattr(rdn, "_launch_stage", counting)
    video = [f.cuda() for f in O.synth_frames(9, B, 48, 80, seed=40 + B, smooth=True)]
    with selection(net, (13, 8, 12)):
        st = StreamingBIN(net)
        seen = []
        for k, f in enumerate(video):
            before, n0 = st.backbone_calls, len(stages)
            got = st.push(f)
            assert (got is None) == (k < 5)
            if got is None:
                continue
            assert st.backbone_calls - before == (13 if k == 5 else 10)
            assert stages[n0:] == [(2, 4 if k == 5 else 1, B), (3, 5, B), (5, 3, B), (5, 1, B)]
            seen.append(got)
        with torch.no_grad():
            for k, got in enumerate(seen):
                ref = net(*video[k:k + 6])
                check_selected(got, ref, (13, 8, 12))
                assert [i for i in range(14) if ref[i] is not None] == [8, 12, 13]
    with torch.no_grad():
        full = net(*video[3:9])
    check_selected(seen[3], full, (13, 8, 12))
    assert st.push(video[0]) is None and len(st.frames) == 1          # the selection changed: the cache starts over
    n0 = len(stages)
    full_stream = [st.push(f) for f in video[1:6]][-1]
    assert stages[n0:] == [(2, 5, B), (3, 6, B), (5, 4, B), (5, 2, B)] and all(o is not None for o in full_stream)


def test_streaming_stage_counts_for_a_step0_selection(net, monkeypatch):
    """(9,) needs frames 0..4 only: stage 1 runs its four step-0 pairs, then 3, 2 and 1 calls, and no ConvLSTM cell."""
    from bin_b200 import ops, rdn
    from bin_b200.streaming import StreamingBIN
    video = [f.cuda() for f in O.synth_frames(6, 1, 32, 48, seed=12)]
    with torch.no_grad():
        full = net(*video)
    stages, real = [], rdn._launch_stage
    monkeypatch.setattr(rdn, "_launch_stage", lambda m, calls, outs, prec: stages.append(len(calls)) or real(m, calls, outs, prec))
    monkeypatch.setattr(ops, "convlstm_group", lambda *a, **k: pytest.fail("a ConvLSTM cell ran"))
    with selection(net, (9,), unwanted="zeros"):
        st = StreamingBIN(net)
        got = [st.push(f) for f in video][-1]
    check_selected(got, full, (9,), "zeros")
    assert stages == STAGE_CALLS[(9,)] and st.backbone_calls == 10


@pytest.mark.parametrize("precision", ["fp16", "fp32"])
def test_self_ensemble_with_a_selection(net, precision):
    frames = [f.cuda() for f in O.synth_frames(6, 2, 34, 50, seed=21, smooth=True)]
    with torch.no_grad():
        with selection(net, None, precision=precision, ensemble="flipx4"):
            full = net(*frames)
        for wanted, unwanted in [((13, 8, 12), "none"), ((9,), "zeros")]:
            with selection(net, wanted, unwanted, precision, ensemble="flipx4"):
                got = net(*frames)
            check_selected(got, full, wanted, unwanted)


def test_streaming_ensemble_with_a_selection(net):
    from bin_b200.streaming import StreamingBIN
    video = [f.cuda() for f in O.synth_frames(7, 1, 48, 80, seed=33, smooth=True)]
    with torch.no_grad():
        with selection(net, None, ensemble="flipx4"):
            full = [net(*video[k:k + 6]) for k in range(2)]
    with selection(net, (13, 8, 12), "zeros", ensemble="flipx4"):
        st = StreamingBIN(net)
        got = [st.push(f) for f in video][5:]
    for g, f in zip(got, full):
        check_selected(g, f, (13, 8, 12), "zeros")
    assert st.backbone_calls == 13 + 10


def test_grad_enabled_call_raises(net):
    from bin_b200 import BinB200Error
    frames = [f.cuda() for f in O.synth_frames(6, 1, 16, 16)]
    with selection(net, (13, 8, 12)):
        with pytest.raises(BinB200Error, match="inference-only"):
            net(*frames)                                  # parameters require grad
        with pytest.raises(BinB200Error, match="set_outputs"):
            net(*[f.clone().requires_grad_(True) for f in frames])


def test_caller_sequence_writes_the_same_three_images():
    """test.py's loop body through the DataParallel wrapper, with (13, 8, 12) and unwanted="zeros" as the shim sets it:
    the three images it writes are the full window's, and Ft_p[7], Ft_p[9] still convert to images."""
    from caller_harness import CallerModel, run_test_py_window, tensor2img
    from bin_b200 import rdn
    model = CallerModel(rdn.bin_stage4_lstm(), "cuda:0", device_ids=[0])
    model.load_state_dict_like_load_network({"InterpNet." + k: v for k, v in O.synth_state_dict(0).items()})
    frames = [f[0] for f in O.synth_frames(6, 1, 90, 160, seed=77, smooth=True)]        # (3,H,W) like read_image
    full_imgs, full, _ = run_test_py_window(model, frames)
    rdn.set_outputs(model.netG, (13, 8, 12), unwanted="zeros")
    imgs, Ft_p, _ = run_test_py_window(model, frames)
    assert all(np.array_equal(a, b) for a, b in zip(imgs, full_imgs))
    check_selected(Ft_p, full, (13, 8, 12), "zeros")
    for k in (7, 9):                                                                     # test.py:399-400
        assert not tensor2img(Ft_p[k].squeeze(0)).any()


def test_full_size_768x1344(monkeypatch):
    from bin_b200 import rdn
    monkeypatch.setenv("BIN_B200_GRAPH", "0")        # eager: one workspace, no graph pool beside it
    net = _new_net()
    try:
        frames = [f.cuda() for f in O.synth_frames(6, 1, 768, 1344, seed=9, smooth=True)]
        with torch.no_grad():
            full = net(*frames)
            rdn.set_outputs(net, (13, 8, 12))
            got = net(*frames)
        check_selected(got, full, (13, 8, 12))
    finally:
        del net
        rdn.release_workspaces()
        torch.cuda.empty_cache()
