"""stream_video on the GPU: every window of a video in test.py's order, edge windows included, bit-identical to calling
the net on that window's clamped frames, in every inference mode and on a light (G0 = 64, D = 6) window; the backbone
calls it counts and launches against its plan; when each window comes out; and the refusals."""
from contextlib import contextmanager

import pytest
import torch

from oracle import arch_oracle as A
from oracle import bin_oracle as O

pytestmark = pytest.mark.gpu
NS = [2, 3, 4, 5, 6, 7, 9]
MODES = ["plain", "selection", "selection-zeros", "flipx4", "fp32", "light"]


@pytest.fixture(scope="module")
def nets():
    from bin_b200 import rdn
    net = rdn.bin_stage4_lstm()
    net.load_state_dict(O.synth_state_dict(0), strict=True)
    light = rdn.bin_stage4_lstm()
    light.model = rdn.RDN_residual_interp_5_input(lstm=True, GO=64, D=6)
    light.load_state_dict(A.synth_state_dict(0, 64, 6), strict=True)
    return {"shipped": net.cuda().eval(), "light": light.cuda().eval()}


@contextmanager
def mode(nets, name):
    from bin_b200 import rdn
    net = nets["light" if name == "light" else "shipped"]
    if name.startswith("selection"):
        rdn.set_outputs(net, (13, 8, 12), "zeros" if name.endswith("zeros") else "none")
    rdn.set_self_ensemble(net, "flipx4" if name == "flipx4" else None)
    rdn.set_precision(net, "fp32" if name == "fp32" else "fp16")
    try:
        yield net
    finally:
        rdn.set_outputs(net, None)
        rdn.set_self_ensemble(net, None)
        rdn.set_precision(net, "fp16")


def planned_calls(net, n):
    from bin_b200 import rdn
    from bin_b200.streaming import VideoPlan
    sel = rdn._outputs_of(net)
    plan = VideoPlan(rdn._window_live(range(14) if sel is None else sel[0]))
    steps = [s for _ in range(n) for s in plan.arrive()] + plan.end()
    return sum(s.backbone_calls for s in steps)


def same(a, b):
    return (a is None and b is None) or (a is not None and b is not None and a.shape == b.shape and torch.equal(a, b))


@pytest.mark.parametrize("name", MODES)
@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("n", NS)
def test_every_window_matches_the_net_on_its_clamped_frames(nets, monkeypatch, n, B, name):
    from bin_b200 import rdn
    from bin_b200.streaming import stream_video, test_py_window
    video = [f.cuda() for f in O.synth_frames(n, B, 32, 48, seed=100 * n + B, smooth=True)]
    launched, real = [], rdn._launch_stage
    monkeypatch.setattr(rdn, "_launch_stage",
                        lambda m, calls, outs, prec: launched.append(len(calls)) or real(m, calls, outs, prec))
    drawn, at = [], []

    def source():                                   # a generator: the stream cannot know N in advance
        for k, f in enumerate(video):
            drawn.append(k)
            yield f

    with mode(nets, name) as net:
        stream = stream_video(net, source())
        got = []
        for i, outs in stream:
            got.append((i, outs))
            at.append(len(drawn))
        stream_launched = sum(launched)
        assert [i for i, _ in got] == list(range(n - 1))
        assert at == [min(i + 4, n) for i in range(n - 1)]         # window i as soon as frame i+3 is there
        assert stream.backbone_calls == planned_calls(net, n) == stream_launched
        if name in ("plain", "fp32", "light"):
            assert stream.backbone_calls == 13 * n - 11
        with torch.no_grad():
            for i, outs in got:
                ref = net(*[video[j] for j in test_py_window(i, n)])
                assert isinstance(outs, tuple) and len(outs) == 14
                assert all(same(a, b) for a, b in zip(outs, ref)), (i, [k for k in range(14) if not same(outs[k], ref[k])])
                assert not any(o is not None and o.requires_grad for o in outs)
    net.__dict__.pop("_graph_entry", None)


def test_edge_window_runs_a_repeated_pair_once(nets, monkeypatch):
    """Window 0 of a 7-frame video reads the pair of frames 0, 0 at two positions: stage 1 runs 4 calls, not 5, and
    every later stage-1 launch runs the one new pair (none for the last window)."""
    from bin_b200 import rdn
    from bin_b200.streaming import stream_video
    video = [f.cuda() for f in O.synth_frames(7, 1, 32, 48, seed=5)]
    stages, real = [], rdn._launch_stage
    monkeypatch.setattr(rdn, "_launch_stage",
                        lambda m, calls, outs, prec: stages.append((m.NFRAMES, len(calls))) or real(m, calls, outs, prec))
    list(stream_video(nets["shipped"], video))
    stage1 = [k for nf, k in stages if nf == 2]
    assert stage1 == [4, 1, 1, 1, 1] and len(stages) == 5 + 3 * 6


@pytest.mark.parametrize("n", [0, 1])
def test_a_video_of_fewer_than_two_frames_has_no_window(nets, n):
    from bin_b200.streaming import stream_video
    stream = stream_video(nets["shipped"], [f.cuda() for f in O.synth_frames(n, 1, 16, 16)])
    assert list(stream) == [] and stream.backbone_calls == 0


def test_refusals(nets):
    from bin_b200 import BinB200Error, rdn
    from bin_b200.streaming import stream_video
    net = nets["shipped"]
    video = [f.cuda() for f in O.synth_frames(5, 1, 16, 16)]
    with pytest.raises(BinB200Error, match="fp32 CUDA frames"):
        list(stream_video(net, [video[0].cpu()]))
    with pytest.raises(BinB200Error, match="first frame"):
        list(stream_video(net, video[:2] + [torch.zeros(1, 3, 16, 18, device="cuda")]))
    stream = stream_video(net, video)
    next(stream)
    try:
        rdn.set_precision(net, "fp32")
        with pytest.raises(BinB200Error, match="changed during the video"):
            next(stream)
    finally:
        rdn.set_precision(net, "fp16")
