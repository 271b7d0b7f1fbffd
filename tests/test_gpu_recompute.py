"""Activation recomputation (rdn.set_activation_checkpointing(net, "recompute")): the same training computations as the
default saving mode, with less memory held between the forward and the backward.

Every value the default mode reproduces bit for bit from run to run is compared with torch.equal: the 14 outputs, every
frame gradient and the weight gradient of every backbone conv.  Three reductions of the existing kernels add partial
sums with float atomicAdd across blocks, so their last bits depend on the order blocks finish, in either mode and from
one run to the next: the pixel-loss terms (bin_pixel_loss_fwd), the backbone bias gradients (db of the backward) and
the ConvLSTM weight and bias gradients (bin_convlstm_bwd).  Those are compared within a few float32 ulps of their
scale (REL)."""
import pytest
import torch

from oracle import bin_oracle as O

pytestmark = pytest.mark.gpu
MODES = (None, "recompute")
REL = 1e-5


def _atomic_sum(name: str) -> bool:
    """Gradients that existing kernels reduce with float atomics (see the module docstring)."""
    return name.endswith(".bias") or ".Gates." in name


def _close(a, b, rel=REL):
    return (a - b).abs().max().item() <= rel * max(a.abs().max().item(), 1e-30)


@pytest.fixture(scope="module")
def net():
    from bin_b200 import rdn
    m = rdn.bin_stage4_lstm()
    m.load_state_dict(O.synth_state_dict(0), strict=True)
    m = m.cuda().train()
    yield m
    rdn.set_activation_checkpointing(m, None)


def _run(net, mode, call, frames, gts, cycle_pairs=None):
    """One forward + fused pixel loss + backward in `mode`; returns everything the two modes must share."""
    from bin_b200 import rdn
    from bin_b200.loss import pixel_loss
    rdn.set_activation_checkpointing(net, mode)
    net.zero_grad(set_to_none=True)
    fr = [f.clone().requires_grad_(True) for f in frames]
    outs = call(fr)
    outs = list(outs) if isinstance(outs, (tuple, list)) else [outs]
    loss, ll = pixel_loss(outs, gts[:len(outs)], "l1", cycle_pairs=cycle_pairs)
    terms = ll[0]._base if ll[0]._base is not None else torch.stack(ll)          # every pair term, cycle terms included
    loss.backward()
    torch.cuda.synchronize()
    grads = {k: (None if p.grad is None else p.grad.clone()) for k, p in net.named_parameters()}
    return ([o.detach().clone() for o in outs], loss.detach().clone(), terms.detach().clone(), grads,
            [f.grad.clone() for f in fr])


def _assert_identical(a, b):
    outs_a, loss_a, terms_a, grads_a, fgrads_a = a
    outs_b, loss_b, terms_b, grads_b, fgrads_b = b
    assert len(outs_a) == len(outs_b)
    for k, (x, y) in enumerate(zip(outs_a, outs_b)):
        assert torch.equal(x, y), ("output", k, (x - y).abs().max().item())
    assert _close(loss_a, loss_b, 1e-6), (loss_a.item(), loss_b.item())
    assert _close(terms_a, terms_b, 1e-6), (terms_a, terms_b)
    assert list(grads_a) == list(grads_b) and len(grads_a) == 540
    assert [k for k in grads_a if grads_a[k] is None] == [k for k in grads_b if grads_b[k] is None]
    live = [k for k in grads_a if grads_a[k] is not None]
    bad = [k for k in live if not _atomic_sum(k) and not torch.equal(grads_a[k], grads_b[k])]
    assert not bad, bad[:8]
    bad = [k for k in live if _atomic_sum(k) and not _close(grads_a[k], grads_b[k])]
    assert not bad, bad[:8]
    assert sum(not _atomic_sum(k) for k in live) >= 66                    # at least one backbone's conv weights
    for k, (x, y) in enumerate(zip(fgrads_a, fgrads_b)):
        assert torch.equal(x, y), ("frame grad", k, (x - y).abs().max().item())
    return grads_a


@pytest.mark.parametrize("B,H,W", [(2, 64, 96), (1, 70, 134)])
def test_window_step_matches_default(net, B, H, W):
    fr = [f.cuda() for f in O.synth_frames(6, B, H, W, seed=71, smooth=True)]
    gt = [f.cuda() for f in O.synth_frames(14, B, H, W, seed=72, smooth=True)]
    res = [_run(net, mode, lambda f: net(*f), fr, gt) for mode in MODES]
    assert res[0][2].numel() == 17
    grads = _assert_identical(*res)
    assert all(g is not None for g in grads.values())                         # the window reaches every parameter


def test_pyramid3_matches_default(net):
    B, H, W = 1, 70, 134
    fr = [f.cuda() for f in O.synth_frames(4, B, H, W, seed=73, smooth=True)]
    gt = [f.cuda() for f in O.synth_frames(6, B, H, W, seed=74, smooth=True)]
    res = [_run(net, mode, lambda f: net.forward_pyramid3(*f), fr, gt, cycle_pairs=()) for mode in MODES]
    grads = _assert_identical(*res)
    assert grads["model.model3_1.UPNet.2.weight"] is not None and grads["model.model4_1.UPNet.2.weight"] is None


def test_pyramid_5_input_matches_default(net):
    B, H, W = 2, 48, 64
    fr = [f.cuda() for f in O.synth_frames(5, B, H, W, seed=75, smooth=True)]
    gt = [f.cuda() for f in O.synth_frames(10, B, H, W, seed=76, smooth=True)]
    res = [_run(net, mode, lambda f: net.model(*f), fr, gt, cycle_pairs=()) for mode in MODES]
    _assert_identical(*res)


def test_single_backbone_matches_default(net):
    B, H, W = 3, 38, 70
    fr = [f.cuda() for f in O.synth_frames(2, B, H, W, seed=77, smooth=True)]
    gt = [f.cuda() for f in O.synth_frames(1, B, H, W, seed=78, smooth=True)]
    res = [_run(net, mode, lambda f: net.model.model1_1(*f), fr, gt, cycle_pairs=()) for mode in MODES]
    grads = _assert_identical(*res)
    assert grads["model.model1_1.RDBs.11.convs.3.conv.0.weight"] is not None
    assert grads["model.model2_1.SFENet1.weight"] is None


def test_three_adam_steps_match():
    """Three optimizer steps per mode from the same weights and batch: each step re-keys the packed-weight caches that
    the recomputing backward packs from, so a stale cache would show up as a different loss or weight.  The atomically
    reduced gradients feed the steps, so from step 2 on the modes are compared against how far the steps move."""
    from bin_b200 import rdn
    from bin_b200.loss import pixel_loss
    from bin_b200.optim import Adam
    B, H, W = 2, 64, 96
    fr = [f.cuda() for f in O.synth_frames(6, B, H, W, seed=81, smooth=True)]
    gt = [f.cuda() for f in O.synth_frames(14, B, H, W, seed=82, smooth=True)]
    results = []
    s0 = {k: v.cuda() for k, v in O.synth_state_dict(1).items()}
    for mode in MODES:
        m = rdn.bin_stage4_lstm()
        m.load_state_dict(O.synth_state_dict(1), strict=True)
        m = rdn.set_activation_checkpointing(m.cuda().train(), mode)
        opt = Adam(m.parameters(), lr=1e-4, betas=(0.9, 0.99))               # yml :52-55
        losses = []
        for _ in range(3):
            opt.zero_grad(set_to_none=True)
            loss, _ = pixel_loss(m(*fr), gt, "l1")
            loss.backward()
            opt.step()
            losses.append(loss.detach().clone())
        torch.cuda.synchronize()
        results.append((torch.stack(losses), {k: v.clone() for k, v in m.state_dict().items()}))
    (la, sa), (lb, sb) = results
    assert _close(la[0], lb[0], 1e-6), (la, lb)                             # same weights: only the loss sum's order
    moved = (la - la[0]).abs().max().item()
    assert moved > 0 and (la - lb).abs().max().item() <= 1e-3 * moved, (la, lb)
    assert list(sa) == list(sb)
    step = torch.sqrt(sum(((sa[k] - s0[k]) ** 2).sum() for k in sa)).item()
    diff = torch.sqrt(sum(((sa[k] - sb[k]) ** 2).sum() for k in sa)).item()
    assert step > 0 and diff <= 1e-2 * step, (diff, step)


def test_modified_weight_between_forward_and_backward_raises(net):
    from bin_b200 import BinB200Error, rdn
    B, H, W = 1, 32, 48
    fr = [f.cuda() for f in O.synth_frames(6, B, H, W, seed=83)]
    rdn.set_activation_checkpointing(net, "recompute")
    try:
        net.zero_grad(set_to_none=True)
        loss = sum(o.sum() for o in net(*fr))
        w = net.model.model2_1.RDBs[5].convs[2].conv[0].weight
        with torch.no_grad():
            w.mul_(1.0)                                            # same values, new version: still refused
        with pytest.raises(BinB200Error, match="modified in place"):
            loss.backward()
    finally:
        rdn.set_activation_checkpointing(net, None)
        net.zero_grad(set_to_none=True)


def test_retain_graph_second_backward_gives_identical_gradients(net):
    """A recomputing node keeps its inputs, not activations, so a second backward through it recomputes from the same
    frames and weights -- even after later work has reused the shared workspace -- and gives the same gradients
    (within REL for the atomically reduced ones)."""
    from bin_b200 import rdn
    B, H, W = 1, 40, 56
    fr = [f.cuda().requires_grad_(True) for f in O.synth_frames(6, B, H, W, seed=84)]
    cot = [f.cuda() - 0.5 for f in O.synth_frames(14, B, H, W, seed=85)]
    rdn.set_activation_checkpointing(net, "recompute")
    try:
        net.zero_grad(set_to_none=True)
        loss = sum((o * c).sum() for o, c in zip(net(*fr), cot))
        loss.backward(retain_graph=True)
        first = {k: p.grad.clone() for k, p in net.named_parameters()}
        ffirst = [f.grad.clone() for f in fr]
        net.zero_grad(set_to_none=True)
        for f in fr:
            f.grad = None
        with torch.no_grad():                                       # overwrite the shared workspace in between
            net.model.model2_1(*[f.cuda() * 0.5 for f in O.synth_frames(3, 6 * B, H, W, seed=86)])
        loss.backward()
        second = {k: p.grad for k, p in net.named_parameters()}
        assert all(torch.equal(a, f.grad) for a, f in zip(ffirst, fr))
        assert not [k for k in first if not _atomic_sum(k) and not torch.equal(first[k], second[k])]
        assert not [k for k in first if _atomic_sum(k) and not _close(first[k], second[k])]
    finally:
        rdn.set_activation_checkpointing(net, None)


@pytest.fixture(scope="module")
def mem_setup():
    from bin_b200 import rdn
    B, H, W = 4, 256, 256
    m = rdn.bin_stage4_lstm()
    m.load_state_dict(O.synth_state_dict(0), strict=True)
    m = m.cuda().train()
    fr = [f.cuda() for f in O.synth_frames(6, B, H, W, seed=91, smooth=True)]
    gt = [f.cuda() for f in O.synth_frames(14, B, H, W, seed=92, smooth=True)]
    yield m, fr, gt, (B, H, W)
    del m, fr, gt
    rdn.release_workspaces()
    torch.cuda.empty_cache()


def test_recompute_peak_memory(mem_setup):
    """Peak memory of a B = 4 x 256x256 window step falls by at least half of S, the saved activations of the default
    mode (bin_backbone_train_workspace_bytes of the four stages: 5, 6, 4 and 2 calls)."""
    from bin_b200 import _lib, rdn
    from bin_b200.loss import pixel_loss
    m, fr, gt, (B, H, W) = mem_setup
    L = _lib.lib()
    S = sum(L.bin_backbone_train_workspace_bytes(n, B * calls, H, W) for n, calls in ((2, 5), (3, 6), (5, 4), (5, 2)))

    def step():
        m.zero_grad(set_to_none=True)
        loss, _ = pixel_loss(m(*fr), gt, "l1")
        loss.backward()
        return loss.detach()

    peaks, losses = {}, {}
    for mode in MODES:
        rdn.release_workspaces()
        rdn.set_activation_checkpointing(m, mode)
        step()                                                       # warm-up: packed caches, the shared workspace
        m.zero_grad(set_to_none=True)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        losses[mode] = step()
        torch.cuda.synchronize()
        peaks[mode] = torch.cuda.max_memory_allocated()
    rdn.set_activation_checkpointing(m, None)
    assert _close(losses[None], losses["recompute"], 1e-6)
    saved = peaks[None] - peaks["recompute"]
    assert saved >= 0.5 * S, (peaks, S, saved / S)
