"""The x4 flip self-ensemble on the GPU: the reference's own flipx4_forward results (tests/golden/ensemble.npz), bit-exact
equality with the same ensemble composed from four plain module calls and torch flips (up to 768x1344, where stage 1
runs at batch 20), the expand / mean kernels against torch.flip, the streaming path, and the refusals."""
import os
from contextlib import contextmanager

import numpy as np
import pytest
import torch

from oracle import bin_oracle as O

pytestmark = pytest.mark.gpu
ORIENTATIONS = [None, (-1,), (-2,), (-2, -1)]          # flipx4_forward's order (utils/test_util.py:119-130)


def _new_net():
    from bin_b200 import rdn
    m = rdn.bin_stage4_lstm()
    m.load_state_dict(O.synth_state_dict(0), strict=True)
    return m.cuda().eval()


@pytest.fixture(scope="module")
def net():
    return _new_net()


@contextmanager
def mode(net, ensemble, precision="fp16"):
    from bin_b200 import rdn
    rdn.set_self_ensemble(net, ensemble)
    rdn.set_precision(net, precision)
    try:
        yield net
    finally:
        rdn.set_self_ensemble(net, None)
        rdn.set_precision(net, "fp16")


def composed(net, frames):
    """((w(x) + flip(w(flipW x))) + flip(w(flipH x))) + flip(w(flipHW x))) / 4 from four plain calls at batch B."""
    assert getattr(net, "self_ensemble", None) is None
    acc = None
    with torch.no_grad():
        for dims in ORIENTATIONS:
            outs = net(*[f if dims is None else torch.flip(f, dims) for f in frames])
            outs = [o if dims is None else torch.flip(o, dims) for o in outs]
            acc = outs if acc is None else [a + o for a, o in zip(acc, outs)]
    return [a / 4 for a in acc]


def ensemble(net, frames, precision="fp16"):
    with mode(net, "flipx4", precision), torch.no_grad():
        return net(*frames)


@pytest.mark.parametrize("precision,bar", [("fp16", 1e-3), ("fp32", 1e-5)])
def test_matches_the_reference_flipx4_forward(net, golden_dir, precision, bar):
    g = np.load(os.path.join(golden_dir, "ensemble.npz"))
    for tag in ("a", "b"):
        B, H, W, seed = (int(v) for v in g[f"{tag}_meta"])
        frames = [f.cuda() for f in O.synth_frames(6, B, H, W, seed=seed, smooth=True)]
        got = torch.stack(ensemble(net, frames, precision)).cpu()
        ref = torch.from_numpy(g[f"{tag}_out"])
        assert got.shape == ref.shape
        err = (got - ref).abs().max().item()
        assert err <= bar, (tag, precision, err)


@pytest.mark.parametrize("B,H,W,precision", [(1, 48, 80, "fp16"), (2, 34, 50, "fp16"), (1, 40, 56, "fp32")])
def test_bit_exact_composition_small(net, B, H, W, precision):
    frames = [f.cuda() for f in O.synth_frames(6, B, H, W, seed=B * 100 + H, smooth=True)]
    got = ensemble(net, frames, precision)
    with mode(net, None, precision):
        ref = composed(net, frames)
    assert len(got) == 14 and all(g.shape == (B, 3, H, W) for g in got)
    assert all(torch.equal(a, b) for a, b in zip(got, ref))


def test_bit_exact_composition_768x1344(monkeypatch):
    """B = 1 at 768x1344: the ensemble's stage-1 launch has 20 batch items and a ~20 GB backbone workspace."""
    from bin_b200 import rdn
    monkeypatch.setenv("BIN_B200_GRAPH", "0")        # plain calls run eagerly: one workspace, no graph pool beside it
    net = _new_net()
    try:
        frames = [f.cuda() for f in O.synth_frames(6, 1, 768, 1344, seed=9, smooth=True)]
        got = ensemble(net, frames)
        ref = composed(net, frames)
        for k, (a, b) in enumerate(zip(got, ref)):
            assert torch.equal(a, b), (k, (a - b).abs().max().item())
    finally:
        del net
        rdn.release_workspaces()
        torch.cuda.empty_cache()


def _flip4(x):
    return torch.cat([x, torch.flip(x, (-1,)), torch.flip(x, (-2,)), torch.flip(x, (-2, -1))])


@pytest.mark.parametrize("n,B,H,W", [(1, 1, 8, 16), (6, 3, 10, 14), (14, 2, 6, 12), (2, 1, 5, 7), (1, 3, 1, 1)])
def test_expand_and_mean_kernels_match_torch(n, B, H, W):
    from bin_b200 import ops
    gen = torch.Generator(device="cuda").manual_seed(n * 1000 + W)
    xs = [torch.randn((B, 3, H, W), generator=gen, device="cuda") for _ in range(n)]
    keep = [x.clone() for x in xs]
    big = ops.flipx4_expand(xs)
    assert all(torch.equal(b, _flip4(x)) for b, x in zip(big, xs))
    # magnitudes spread over 2^-20..2^20 so that any other summation order changes the bits
    ys = [torch.randn((4 * B, 3, H, W), generator=gen, device="cuda") *
          torch.exp2(torch.randint(-20, 21, (4 * B, 3, H, W), generator=gen, device="cuda").float()) for _ in range(n)]
    means = ops.flipx4_mean(ys)
    for m, y in zip(means, ys):
        y0, y1, y2, y3 = y.chunk(4)
        ref = (((y0 + torch.flip(y1, (-1,))) + torch.flip(y2, (-2,))) + torch.flip(y3, (-2, -1))) / 4
        assert m.shape == (B, 3, H, W) and torch.equal(m, ref)
    assert all(torch.equal(a, b) for a, b in zip(xs, keep))
    # mean(expand(x)) == x exactly: the four copies are equal, and 4x / 4 is exact
    assert all(torch.equal(m, x) for m, x in zip(ops.flipx4_mean(big), xs))


def test_kernels_on_unaligned_tensors():
    """W % 4 == 0 but a tensor 4 bytes off a 16-byte boundary: the kernels take their scalar path."""
    from bin_b200 import ops
    base = torch.randn(2 * 3 * 8 * 16 + 1, device="cuda")
    x = base[1:].view(2, 3, 8, 16)
    assert x.is_contiguous() and x.data_ptr() % 16 != 0
    assert torch.equal(ops.flipx4_expand([x])[0], _flip4(x))
    ybase = torch.randn(8 * 3 * 8 * 16 + 1, device="cuda")
    y = ybase[1:].view(8, 3, 8, 16)
    y0, y1, y2, y3 = y.chunk(4)
    ref = (((y0 + torch.flip(y1, (-1,))) + torch.flip(y2, (-2,))) + torch.flip(y3, (-2, -1))) / 4
    assert torch.equal(ops.flipx4_mean([y])[0], ref)


@pytest.mark.parametrize("B", [1, 2])
def test_streaming_is_bit_identical_to_window_calls(net, B):
    from bin_b200.streaming import StreamingBIN
    video = [f.cuda() for f in O.synth_frames(8, B, 48, 80, seed=31 + B, smooth=True)]
    with mode(net, "flipx4"):
        st = StreamingBIN(net)
        got = [st.push(f) for f in video]
        assert all(g is None for g in got[:5]) and all(g is not None for g in got[5:])
        with torch.no_grad():
            for k in range(3):
                ref = net(*video[k:k + 6])
                assert all(torch.equal(a, b) for a, b in zip(got[5 + k], ref)), k
                assert all(a.shape == (B, 3, 48, 80) for a in got[5 + k])
        assert st.backbone_calls == 17 + 2 * 13
    plain_next = st.push(video[0])                        # the mode changed: the cache starts over
    assert plain_next is None and len(st.frames) == 1 and st.frames[0][1].shape == (B, 3, 48, 80)


def test_inputs_unmutated_and_plain_calls_unchanged(net):
    frames = [f.cuda() for f in O.synth_frames(6, 1, 32, 48, seed=5)]
    keep = [f.clone() for f in frames]
    with torch.no_grad():
        before = net(*frames)
    ens = ensemble(net, frames)
    assert all(torch.equal(a, b) for a, b in zip(frames, keep))
    with torch.no_grad():
        after = net(*frames)
    assert all(torch.equal(a, b) for a, b in zip(before, after))
    assert not all(torch.equal(a, b) for a, b in zip(before, ens))
    assert len({o.data_ptr() for o in ens}) == 14 and all(o.is_contiguous() for o in ens)


def test_grad_enabled_and_pyramid3_calls_raise(net):
    from bin_b200 import BinB200Error
    frames = [f.cuda() for f in O.synth_frames(6, 1, 16, 16)]
    with mode(net, "flipx4"):
        with pytest.raises(BinB200Error, match="inference-only"):
            net(*frames)                                  # parameters require grad
        with torch.no_grad(), pytest.raises(BinB200Error, match="forward_pyramid3"):
            net.forward_pyramid3(*frames[:4])
        with pytest.raises(BinB200Error, match="inference-only"):
            net(*[f.requires_grad_(True) for f in frames])
