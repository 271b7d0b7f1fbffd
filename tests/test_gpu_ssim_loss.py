"""The fused SSIM loss (ssim_loss.cu, `loss.ssim`, `pixel_loss(..., "cb+ssim")`, DESIGN §4r) on the GPU: the forward
and both gradients against the fp64 oracle (oracle/ssim_oracle.py, pinned to the reference's utils/util.py), the
17-term criterion against its parts, determinism, and the training driver with the criterion: graph against eager,
the driver against a hand-written loop, validation, and no host synchronisation."""
import os
import random
import statistics
import subprocess
import sys

import pytest
import torch

from oracle import bin_oracle as O
from oracle import ssim_oracle as S

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = 2.0 ** -24                  # fp32 unit roundoff
FWD_ERRS = []                   # (case, err, bar) of every forward case, summarised by the last forward test


def _images(kind, B, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    r = lambda: torch.rand(B, 3, h, w, generator=g, dtype=torch.float64)
    if kind == "unit":                                       # [0, 1], mostly independent
        a = r()
        return a, 0.4 * a + 0.6 * r()
    if kind == "wide":                                       # out to 0.5 beyond [0, 1]
        a = r() * 2 - 0.5
        return a, (a + 0.2 * (r() - 0.5)).clamp(-0.5, 1.5)
    if kind == "smooth":                                     # photograph-like, small residual: high SSIM
        k = torch.ones(1, 1, 5, 5, dtype=torch.float64) / 25
        a = torch.nn.functional.conv2d(r().reshape(-1, 1, h, w), k, padding=2).reshape(B, 3, h, w)
        return a, a + 0.01 * (r() - 0.5)
    if kind == "identical":
        a = r()
        return a, a.clone()
    if kind == "constant":                                   # sigma = 0 in both
        return torch.full((B, 3, h, w), 0.25, dtype=torch.float64), torch.full((B, 3, h, w), 0.75, dtype=torch.float64)
    raise ValueError(kind)


def _f32(*ts):
    return [t.float().cuda() for t in ts]


def _derivative_maps(a, b):
    """fp64 SSIM map and its derivatives w.r.t. the raw filtered moments G*a, G*b, G*a^2, G*b^2, G*ab."""
    mom = [S._filt(t).detach().requires_grad_() for t in (a, b, a * a, b * b, a * b)]
    ma, mb, saa, sbb, sab = mom
    A1, A2 = 2 * ma * mb + S.C1, 2 * (sab - ma * mb) + S.C2
    B1, B2 = ma * ma + mb * mb + S.C1, (saa - ma * ma) + (sbb - mb * mb) + S.C2
    smap = (A1 * A2) / (B1 * B2)
    smap.sum().backward()
    return smap.detach(), [m.grad for m in mom]


def _fwd_bar(a, b):
    """Bound on |fp32 mean SSIM - fp64 mean SSIM|.  Each filtered moment is 22 fp32 multiply-adds over terms of size
    <= M^2 (M = max(1, max |x|)): its error is at most delta = 24 u M^2.  The variance cancellation G*a^2 - (G*a)^2
    turns that into an error of S weighted by the derivative of S with respect to each raw moment, so a position's
    bar is delta * sum |dS/dmoment| plus the rounding of the map's own few operations; the mean adds the tile and
    pair summation."""
    M = max(1.0, a.abs().max().item(), b.abs().max().item())
    smap, d = _derivative_maps(a, b)
    per = 24 * U * M * M * sum(x.abs() for x in d) + 8 * U * smap.abs()
    return per.mean().item() + 32 * U * smap.abs().mean().item()


FWD_CASES = [(1, 11, 11), (2, 12, 13), (3, 37, 53), (2, 128, 256), (3, 256, 256)]   # 3 x 256^2: 576 tiles > 132 SMs


@pytest.mark.parametrize("kind", ["unit", "wide", "smooth", "identical", "constant"])
@pytest.mark.parametrize("B,h,w", FWD_CASES)
def test_forward_against_fp64(B, h, w, kind):
    from bin_b200.loss import ssim
    a, b = _images(kind, B, h, w, seed=B * 1000 + h + w)
    a, b = [t.float().double() for t in (a, b)]              # the values the fp32 kernel sees
    got = ssim(*_f32(a, b)).item()
    want = S.ssim(a, b).item()
    bar = _fwd_bar(a, b)
    err = abs(got - want)
    FWD_ERRS.append((f"{kind} {B}x{h}x{w}", err, bar))
    print(f"ssim fwd {kind:9s} B={B} {h}x{w}: got {got:.9f} want {want:.9f} err {err:.3e} bar {bar:.3e} "
          f"err/bar {err / bar:.3f}")
    assert err <= bar
    if kind == "identical":
        assert abs(got - 1.0) <= bar


def test_forward_error_summary():
    """Runs after the forward cases (file order): the worst and the median err/bar, as DESIGN §4r quotes them."""
    if not FWD_ERRS:
        pytest.skip("run with the forward cases")
    ratios = [e / b for _, e, b in FWD_ERRS]
    worst = max(range(len(ratios)), key=ratios.__getitem__)
    print(f"ssim fwd summary: {len(ratios)} cases, worst err/bar {ratios[worst]:.3f} ({FWD_ERRS[worst][0]}), "
          f"median err/bar {statistics.median(ratios):.3f}, worst err {max(e for _, e, _ in FWD_ERRS):.3e}")


def _full(m):
    """G (*) m: the full correlation of (B, C, h-10, w-10) maps with the 11 x 11 window -> (B, C, h, w)."""
    g = torch.tensor(S.GAUSS11, dtype=m.dtype)
    n, c, hv, wv = m.shape
    k = torch.outer(g, g).view(1, 1, 11, 11)
    return torch.nn.functional.conv_transpose2d(m.reshape(n * c, 1, hv, wv), k).reshape(n, c, hv + 10, wv + 10)


def _grad_scale(a, b):
    """Per element of (dSum/da, dSum/db): the sum of the magnitudes of the terms the backward adds,
    G(*)|alpha| + 2|a| G(*)|beta| + |b| G(*)|gamma|.  The maps' worst relative error is the forward's cancellation in
    s_aa + s_bb + C2 >= C2: 2 delta / C2 with delta = 24 u M^2, and the full correlation adds a few u."""
    _, (da_, db_, daa, dbb, dab) = _derivative_maps(a, b)
    fb, fg = _full(daa.abs()), _full(dab.abs())
    return _full(da_.abs()) + 2 * a.abs() * fb + b.abs() * fg, _full(db_.abs()) + 2 * b.abs() * fb + a.abs() * fg


def _rel_bar(a, b):
    M = max(1.0, a.abs().max().item(), b.abs().max().item())
    return 64 * U * M * M / S.C2


@pytest.mark.parametrize("kind", ["unit", "wide", "smooth", "identical"])
@pytest.mark.parametrize("B,h,w", [(1, 11, 11), (2, 12, 13), (3, 37, 53), (2, 128, 256)])
def test_backward_against_fp64(B, h, w, kind):
    from bin_b200.loss import ssim
    a, b = [t.float().double() for t in _images(kind, B, h, w, seed=7 * B + h * w)]
    ga, gb = [t.requires_grad_() for t in _f32(a, b)]
    ssim(ga, gb).backward()
    ra, rb = [t.clone().requires_grad_() for t in (a, b)]
    S.ssim(ra, rb).backward()
    n = B * 3 * (h - 10) * (w - 10)
    sa, sb = _grad_scale(a, b)
    rel = _rel_bar(a, b)
    for name, got, want, sc in (("da", ga.grad, ra.grad, sa), ("db", gb.grad, rb.grad, sb)):
        err = (got.double().cpu() - want).abs()
        bar = rel * sc / n + 8 * U * want.abs()
        gmax = want.abs().max().item()
        print(f"ssim bwd {kind:9s} B={B} {h}x{w} {name}: max err {err.max().item():.3e}, max|grad| {gmax:.3e}, "
              f"err/max|grad| {err.max().item() / gmax:.3e}, worst err/bar {(err / bar).max().item():.3f}")
        assert (err <= bar).all(), name


def _outs_gts(B, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    outs = [torch.rand(B, 3, h, w, generator=g, dtype=torch.float64) * 1.2 - 0.1 for _ in range(14)]
    gts = [(o + 0.2 * (torch.rand(B, 3, h, w, generator=g, dtype=torch.float64) - 0.5)).clamp(0, 1) for o in outs]
    return [o.float().double() for o in outs], [t.float().double() for t in gts]


def test_cb_ssim_gradients_through_the_cycle_terms():
    """pixel_loss('cb+ssim') over the 14 terms and the cycle pairs (1,7), (5,9), (2,8): outputs 1, 2, 5, 7, 8 and 9
    each feed two terms.  Per tensor against fp64 autograd of the oracle criterion."""
    from bin_b200.loss import CYCLE_PAIRS_6V2, pixel_loss
    B, h, w, wt = 2, 24, 40, 0.5
    outs, gts = _outs_gts(B, h, w, seed=5)
    go = [t.float().cuda().requires_grad_() for t in outs]
    loss, lst = pixel_loss(go, [t.float().cuda() for t in gts], "cb+ssim", ssim_weight=wt)
    loss.backward()
    ro = [t.clone().requires_grad_() for t in outs]
    rloss, rterms = S.cb_ssim_loss(ro, gts, wt)
    rloss.backward()
    assert abs(loss.item() - rloss.item()) <= 1e-5 * abs(rloss.item())
    for k in range(14):
        assert abs(lst[k].item() - rterms[k].item()) <= 1e-5 * abs(rterms[k].item())
    # bar per output: the SSIM backward's bound of every term it feeds, plus fp32 rounding of the Charbonnier part
    pairs = [(k, None) for k in range(14)] + list(CYCLE_PAIRS_6V2)
    n = B * 3 * (h - 10) * (w - 10)
    scale = [torch.zeros_like(t) for t in outs]
    uses = [0] * 14
    rel = 0.0
    for k, (i, j) in enumerate(pairs):
        x, y = outs[i], (gts[i] if j is None else outs[j])
        sx, sy = _grad_scale(x, y)
        scale[i] += sx * wt / (17 * n)
        uses[i] += 1
        if j is not None:
            scale[j] += sy * wt / (17 * n)
            uses[j] += 1
        rel = max(rel, _rel_bar(x, y))
    numel = B * 3 * h * w
    for k in range(14):
        err = (go[k].grad.double().cpu() - ro[k].grad).abs()
        # the Charbonnier gradient of each term is at most 1 / (17 numel) per element, rounded a few times
        bar = rel * scale[k] + 16 * U * ro[k].grad.abs() + 8 * U * uses[k] / (17 * numel)
        print(f"cb+ssim grad of output {k:2d}: max err {err.max().item():.3e}, max|grad| "
              f"{ro[k].grad.abs().max().item():.3e}, worst err/bar {(err / bar).max().item():.3f}")
        assert (err <= bar).all(), k


def test_whole_loss_is_cb_plus_weighted_ssim():
    from bin_b200.loss import CYCLE_PAIRS_6V2, pixel_loss, ssim
    torch.use_deterministic_algorithms(True)
    try:
        outs, gts = _outs_gts(2, 40, 56, seed=11)
        outs, gts = [t.float().cuda() for t in outs], [t.float().cuda() for t in gts]
        wt = 0.01
        total, lst = pixel_loss(outs, gts, "cb+ssim", ssim_weight=wt)
        _, cb = pixel_loss(outs, gts, "cb")
        cb_all = cb[0]._base                                 # all 17 Charbonnier terms
        pairs = list(zip(outs, gts)) + [(outs[i], outs[j]) for i, j in CYCLE_PAIRS_6V2]
        want = torch.stack([cb_all[k] + wt * (1.0 - ssim(x, y)) for k, (x, y) in enumerate(pairs)])
        got = lst[0]._base
        assert got.shape == (17,)
        assert torch.allclose(got, want, rtol=4 * U, atol=0)
        assert abs(total.item() - want.sum().item() / 17) <= 8 * U * abs(total.item())
        print(f"cb+ssim terms vs cb + w (1 - ssim): bitwise equal {torch.equal(got, want)}, max diff "
              f"{(got - want).abs().max().item():.3e}")
    finally:
        torch.use_deterministic_algorithms(False)


_CHILD = r"""
import hashlib, sys
sys.path.insert(0, %r)
import torch
from bin_b200.loss import pixel_loss
torch.use_deterministic_algorithms(True)
g = torch.Generator().manual_seed(3)
outs = [(torch.rand(2, 3, 128, 256, generator=g) * 1.2 - 0.1).cuda().requires_grad_() for _ in range(14)]
gts = [torch.rand(2, 3, 128, 256, generator=g).cuda() for _ in range(14)]
h = lambda ts: hashlib.sha256(b"".join(t.detach().cpu().numpy().tobytes() for t in ts)).hexdigest()
for rep in range(2):
    for o in outs:
        o.grad = None
    loss, lst = pixel_loss(outs, gts, "cb+ssim", ssim_weight=0.01)
    loss.backward()
    print("LOSS", h([loss] + lst))
    print("GRADS", h([o.grad for o in outs]))
"""


def test_bits_do_not_depend_on_the_run_or_the_sm_count():
    got = {}
    for tag in ("all", "66"):
        env = {k: v for k, v in os.environ.items() if k != "BIN_B200_MAX_SMS"}
        if tag != "all":
            env["BIN_B200_MAX_SMS"] = tag
        r = subprocess.run([sys.executable, "-c", _CHILD % ROOT], env=env, capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, (tag, r.stderr[-3000:])
        lines = r.stdout.strip().splitlines()
        assert len(lines) == 4 and lines[:2] == lines[2:], (tag, lines)         # two runs in one process
        got[tag] = lines[:2]
    assert got["all"] == got["66"], got


# ----------------------------------------------------------------------------- the training driver
def _opts(root, save, weights, **over):
    from test_gpu_train_driver import options
    kw = {"train.pixel_criterion": "cb+ssim", "train.ssim_weight": 0.01}
    kw.update(over)
    return options(root, save, weights, **kw)


def _driver(opt, iters, **kw):
    from bin_b200 import train as T
    t = T.Trainer(T.parse_options(opt), deterministic=True, stdout=False, **kw)
    try:
        t.run(max_iters=iters)
    finally:
        t.close()
    return t


@pytest.fixture(scope="module")
def data(tmp_path_factory):
    from test_gpu_train_driver import make_tree
    root = tmp_path_factory.mktemp("ssim_tree")
    tree = str(root / "blur")
    make_tree(tree, "train", ["clipA", "clipB", "clipC"], 1)
    make_tree(tree, "test", ["clipV"], 2)
    w = str(root / "shipped.pth")
    torch.save(O.synth_state_dict(0), w)
    return tree, w


@pytest.fixture(autouse=True)
def _restore_determinism():
    yield
    torch.use_deterministic_algorithms(False)
    torch.utils.deterministic.fill_uninitialized_memory = True
    torch.cuda.set_sync_debug_mode(0)


def _log(save):
    log = open(os.path.join(save, "experiments", "bin_test", "train_bin_test.log")).read().splitlines()
    return [line.split(" - ", 1)[1] for line in log if "iter:" in line]


def test_driver_graph_equals_eager(data, tmp_path):
    """7 iterations with a validation and a ReduceLROnPlateau step at 3 and 6 and losses logged every 2; the graphed
    iterations under sync-debug "error"."""
    from test_gpu_train_driver import assert_same_training
    tree, w = data
    over = {"logger.save_checkpoint_freq": 3, "train.val_freq": 3}
    a = _driver(_opts(tree, str(tmp_path / "eager"), w, **over), 7)
    b = _driver(_opts(tree, str(tmp_path / "graph"), w, **over), 7, cuda_graph=True, sync_debug="error")
    assert b.cuda_graph and b._graph is not None and not a.cuda_graph
    assert_same_training(a.net, a.opt, b.net, b.opt)
    la, lb = _log(str(tmp_path / "eager")), _log(str(tmp_path / "graph"))
    assert la == lb and any("Validation" in line for line in la)
    printed = [line for line in la if "ssim_loss:" in line]
    assert len(printed) == 3, la                              # iterations 2, 4 and 6
    assert torch.equal(a.loss_sums, b.loss_sums)


def _hand_loop(root, weights, iters, wt):
    """The INTEGRATION loop with pixel_loss('cb+ssim')."""
    from bin_b200 import rdn
    from bin_b200.evaluate import load_weights
    from bin_b200.loss import pixel_loss
    from bin_b200.optim import Adam
    from bin_b200.trainset import DeviceBINDataset
    from test_gpu_train_driver import SEED, gts
    torch.use_deterministic_algorithms(True)
    torch.utils.deterministic.fill_uninitialized_memory = False
    random.seed(SEED)
    torch.manual_seed(SEED)
    ds = DeviceBINDataset.from_tree(root, mode="train", device="cuda", lq_size=(3, 128, 256))
    net = rdn.bin_stage4_lstm()
    load_weights(net, weights)
    net = net.cuda().train()
    opt = Adam(net.parameters(), lr=1e-4, betas=(0.9, 0.99), weight_decay=0)
    step = 0
    while step < iters:
        for b in ds.batches(range(len(ds)), 2):
            opt.zero_grad(set_to_none=True)
            outs = net(*[b["LQs"][:, k] for k in range(6)])
            loss, _ = pixel_loss(outs, gts(b), "cb+ssim", nframes=6, version=2, ssim_weight=wt)
            (1.0 * loss).backward()
            opt.step()
            step += 1
            if step == iters:
                break
    return net, opt


def test_driver_equals_hand_loop_and_validates_with_the_criterion(data, tmp_path):
    from bin_b200.loss import pixel_loss
    from bin_b200.trainset import DeviceBINDataset
    from test_gpu_train_driver import SEED, assert_same_training, gts
    tree, w = data
    t = _driver(_opts(tree, str(tmp_path), w), 6)
    net, opt = _hand_loop(tree, w, 6, 0.01)
    assert t.step == 6
    assert_same_training(t.net, t.opt, net, opt)
    t.validate()
    vs = DeviceBINDataset.from_tree(tree, mode="test", lq_size=(3, 128, 256), rng=random.Random(SEED))
    vs.rng = random.Random(SEED)
    total = 0.0
    with torch.no_grad():
        for i in range(len(vs)):
            b = vs.batch([i])
            loss, _ = pixel_loss(t.net(*[b["LQs"][:, k] for k in range(6)]), gts(b), "cb+ssim", ssim_weight=0.01)
            total += loss.item()
    assert t.val_sums[14] == total                            # the mean-loss sum ReduceLROnPlateau steps on


def test_ordinary_iterations_do_not_synchronise(data, tmp_path):
    tree, w = data
    t = _driver(_opts(tree, str(tmp_path), w, **{"logger.print_freq": 3}), 6, sync_debug="error")
    assert t.step == 6
    assert sum("ssim_loss:" in line for line in _log(str(tmp_path))) == 2
