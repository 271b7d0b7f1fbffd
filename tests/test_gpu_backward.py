"""Backward parity (BASELINE config 3): gradients from the sm_90a dgrad/wgrad kernels against autograd
through the fp32 CPU oracle (and the reference's own autograd via tests/golden/window_grad.npz).
Gradients travel as loss-scaled fp16 -> tolerance 2 % of the tensor's max magnitude."""
import os

import numpy as np
import pytest
import torch

from oracle import bin_oracle as O

pytestmark = pytest.mark.gpu
REL = 2e-2


def _close(got, ref, rel=REL):
    scale = ref.abs().max().item()
    return (got - ref).abs().max().item() <= rel * max(scale, 1e-12), ((got - ref).abs().max().item(), scale)


@pytest.fixture(scope="module")
def net():
    from bin_b200 import rdn
    m = rdn.bin_stage4_lstm()
    m.load_state_dict(O.synth_state_dict(0), strict=True)
    return m.cuda()


def _oracle_backbone_grads(name, n, B, H, W, sd):
    bsd = {k: v.clone().requires_grad_(True) for k, v in O.sub_sd(sd, "model." + name).items()}
    fr = [f.requires_grad_(True) for f in O.synth_frames(n, B, H, W, seed=41)]
    cot = O.synth_frames(1, B, H, W, seed=42)[0] - 0.5
    y = O.backbone(fr, bsd)
    loss = (y * cot).sum()
    names = list(bsd.keys())
    grads = torch.autograd.grad(loss, fr + [bsd[k] for k in names])
    return fr, cot, y, grads[:n], dict(zip(names, grads[n:]))


@pytest.mark.parametrize("name,n", [("model1_1", 2), ("model2_1", 3), ("model3_1", 5)])
def test_backbone_backward(net, name, n):
    sd = O.synth_state_dict(0)
    B, H, W = 2, 44, 68          # odd tile remainders in both axes, two batch items
    fr, cot, y_ref, gfr_ref, gp_ref = _oracle_backbone_grads(name, n, B, H, W, sd)
    model = getattr(net.model, name)
    for p in model.parameters():
        p.grad = None
    frames = [f.detach().cuda().requires_grad_(True) for f in fr]
    y = model(*frames)
    assert (y.detach().cpu() - y_ref.detach()).abs().max().item() <= 1e-3
    (y * cot.cuda()).sum().backward()
    for k in range(n):
        ok, info = _close(frames[k].grad.cpu(), gfr_ref[k])
        assert ok, ("frame", k, info)
    got = dict(model.named_parameters())
    bad = []
    for key, ref in gp_ref.items():
        g = got[key].grad
        assert g is not None, key
        ok, info = _close(g.cpu(), ref)
        if not ok:
            # ~750 low-res positions per image: a few ReLU sign flips (fp16 vs fp32 forward) shift single weight grads by
            # several % of the tensor max (1/sqrt(#pixels)); require near-perfect correlation instead
            corr = torch.corrcoef(torch.stack([g.cpu().flatten(), ref.flatten()]))[0, 1].item()
            if not (corr >= 0.997 and info[0] <= 0.15 * info[1]):
                bad.append((key, info, corr))
    assert not bad, bad[:8]


def test_convlstm_backward(net):
    sd = O.synth_state_dict(0)
    g = torch.Generator().manual_seed(3)
    x = torch.rand((2, 3, 12, 14), generator=g)
    c0 = torch.randn((2, 3, 12, 14), generator=g)
    h0 = torch.randn((2, 3, 12, 14), generator=g).tanh()
    cot_h, cot_c = torch.randn((2, 3, 12, 14), generator=g), torch.randn((2, 3, 12, 14), generator=g)
    cell = net.clstm_5_prime_prime
    for state in (None, (c0, h0)):
        lsd = {k: v.clone().requires_grad_(True) for k, v in sd.items() if k.startswith("clstm_5_prime_prime.")}
        xr = x.clone().requires_grad_(True)
        st = None if state is None else tuple(t.clone().requires_grad_(True) for t in state)
        h, (c, _) = O.convlstm(xr, lsd, "clstm_5_prime_prime", st)
        loss = (h * cot_h).sum() + (c * cot_c).sum()
        leaves = [xr, lsd["clstm_5_prime_prime.Gates.weight"], lsd["clstm_5_prime_prime.Gates.bias"]] + (list(st) if st else [])
        ref = torch.autograd.grad(loss, leaves)
        cell.Gates.weight.grad = cell.Gates.bias.grad = None
        xg = x.clone().cuda().requires_grad_(True)
        stg = None if state is None else [t.clone().cuda().requires_grad_(True) for t in state]
        hh, (cc, hh2) = cell(xg, stg)
        ((hh * cot_h.cuda()).sum() + (cc * cot_c.cuda()).sum()).backward()
        got = [xg.grad, cell.Gates.weight.grad, cell.Gates.bias.grad] + ([t.grad for t in stg] if stg else [])
        for a, b in zip(got, ref):
            assert (a.cpu() - b).abs().max().item() <= 1e-4 * max(1.0, b.abs().max().item())


def test_window_backward_vs_reference_autograd(net, golden_dir):
    """d(sum_k <out_k, cot_k>) / d(frames, params) against the REFERENCE's autograd (tests/golden/window_grad.npz)."""
    g = {k: torch.from_numpy(v) for k, v in np.load(os.path.join(golden_dir, "window_grad.npz")).items()}
    net.train()
    net.zero_grad(set_to_none=True)
    fr = [f.cuda().requires_grad_(True) for f in O.synth_frames(6, 1, 16, 16, seed=9)]
    outs = net(*fr)
    cots = O.synth_frames(14, 1, 16, 16, seed=10)
    loss = sum((o * (c.cuda() - 0.5)).sum() for o, c in zip(outs, cots))
    assert abs(loss.item() - g["loss"].item()) <= 2e-2 * max(1.0, abs(g["loss"].item()))
    loss.backward()
    net.eval()
    for k in range(6):
        ref = g[f"dframe{k}"]
        err = (fr[k].grad.cpu() - ref).abs().max().item() / ref.abs().max().item()
        assert err <= 0.05, ("frame", k, err)
    params = dict(net.named_parameters())
    for key in [k[2:] for k in g if k.startswith("d:")]:
        ref = g["d:" + key]
        got = params[key].grad.cpu()
        corr = torch.corrcoef(torch.stack([got.flatten(), ref.flatten()]))[0, 1].item()
        err = (got - ref).abs().max().item() / max(ref.abs().max().item(), 1e-12)
        # 8x8 low-res images: a handful of ReLU sign flips (fp16 vs fp32 forward) move individual weight grads by
        # several % of the tensor max; direction must still agree
        assert corr >= 0.995 and err <= 0.15, (key, corr, err)


@pytest.mark.parametrize("cin,cout,k,split", [(128, 32, 3, 96), (96, 96, 3, None), (224, 96, 1, 96), (36, 96, 5, None),
                                              (96, 256, 3, None), (64, 3, 3, None)])
def test_single_conv_dgrad_wgrad_exact(cin, cout, k, split):
    """One conv, no ReLU: dX (same kernel, transposed weights) and dW (MN-major wgmma GEMM) against autograd of
    F.conv2d on the SAME fp16-rounded operands -> only accumulation-order noise remains (<= 2e-3 of max)."""
    _single_conv_dgrad_wgrad(cin, cout, k, split, 2, 27, 41)


def test_single_conv_wgrad_one_stage_ring():
    """5x5 with 128 < Cout <= 256 leaves room for only ONE wgrad pipeline stage (N = 256); 2 x 64 x 160 is 160 tiles of
    8 x 16, more than one per CTA, so the stage must be recycled inside a CTA."""
    _single_conv_dgrad_wgrad(36, 200, 5, None, 2, 64, 160)


def _single_conv_dgrad_wgrad(cin, cout, k, split, B, H, W):
    import ctypes as C
    import torch.nn.functional as F
    from bin_b200 import _lib, ops
    from bin_b200._lib import Act, check, lib
    torch.manual_seed(1)
    torch.backends.cudnn.allow_tf32 = False          # the fp32 cuDNN reference must not run in TF32
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = "cuda"
    x = torch.randn(B, cin, H, W, device=dev).half().float()
    w = (torch.randn(cout, cin, k, k, device=dev) / (cin * k * k) ** 0.5).half().float()
    dy = torch.randn(B, cout, H, W, device=dev).half().float()
    # fp64 CPU reference (cuDNN's fp32 wgrad was measured 1e-2 off at these shapes; ours agrees with fp64 to 1e-6)
    x64, w64 = x.double().cpu().requires_grad_(True), w.double().cpu().requires_grad_(True)
    gx_ref, gw_ref = torch.autograd.grad((F.conv2d(x64, w64, None, padding=k // 2) * dy.double().cpu()).sum(), [x64, w64])
    gx_ref, gw_ref = gx_ref.float().cuda(), gw_ref.float().cuda()
    st = torch.cuda.current_stream().cuda_stream
    # ---- dgrad
    cin_pad_t, cout_pad_t = (cout + 31) // 32 * 32, (cin + 95) // 96 * 96
    wt = torch.empty(cout_pad_t * cin_pad_t * k * k, dtype=torch.float16, device=dev)
    check(lib().bin_pack_conv_weight_t(w.detach().data_ptr(), cout, cin, k, 0, cin, cout_pad_t, cin_pad_t, wt.data_ptr(), st))
    dyp = ops.nchw_to_p8(dy)
    dx = torch.zeros((B, (cin + 7) // 8, H, W, 8), dtype=torch.float16, device=dev)
    zero_bias = torch.zeros(cout_pad_t, device=dev)
    ops.conv_fwd(dyp, wt, zero_bias, k, cout_pad_t, in0_planes=cin_pad_t // 8, out=dx, store_planes=(cin + 7) // 8)
    torch.cuda.synchronize()
    got = ops.p8_to_nchw(dx, cin)
    assert (got - gx_ref).abs().max().item() <= 2e-3 * gx_ref.abs().max().item()
    # ---- wgrad
    scale = torch.full((1,), 4.0, device=dev)
    dys = ops.nchw_to_p8(dy * 4.0, pad_to=16)                      # the wgrad reads dY planes up to Cout rounded to 16
    dw = torch.zeros_like(w)
    if split is None:
        x0 = ops.nchw_to_p8(x.detach(), pad_to=32)
        x1, x1p = Act(None, 0, 0, 0, 0), 0
        x0p = x0.shape[1]
        a1 = x1
    else:
        x0 = ops.nchw_to_p8(x.detach()[:, :split].contiguous())
        x1t = ops.nchw_to_p8(x.detach()[:, split:].contiguous())
        x0p, x1p = split // 8, (cin - split) // 8
        a1 = ops.act_view(x1t)
    wsp = torch.empty(lib().bin_conv_wgrad_workspace_bytes(), dtype=torch.uint8, device=dev)
    check(lib().bin_conv_wgrad(ops.act_view(x0), 0, x0p, a1, 0, x1p, ops.act_view(dys), 0, cout, cin, k,
                               scale.data_ptr(), dw.data_ptr(), wsp.data_ptr(), st))
    torch.cuda.synchronize()
    assert (dw - gw_ref).abs().max().item() <= 1e-4 * gw_ref.abs().max().item()


def test_pyramid3_training_config3a(net):
    """BASELINE config 3a: fwd+bwd of the 4-frame 3-stage graph; frame gradients vs oracle autograd."""
    sd = O.synth_state_dict(0)
    leaves = {k: v.clone().requires_grad_(True) for k, v in sd.items() if k.startswith("model.model")}
    fr = [f.requires_grad_(True) for f in O.synth_frames(4, 1, 24, 40, seed=5)]
    outs = O.pyramid3_4frames(fr, {**sd, **leaves})
    cots = O.synth_frames(6, 1, 24, 40, seed=6)
    loss = sum((o * (c - 0.5)).sum() for o, c in zip(outs, cots))
    gref = torch.autograd.grad(loss, fr)
    net.zero_grad(set_to_none=True)
    frg = [f.detach().cuda().requires_grad_(True) for f in fr]
    got = net.forward_pyramid3(*frg)
    sum((o * (c.cuda() - 0.5)).sum() for o, c in zip(got, cots)).backward()
    for k in range(4):
        err = (frg[k].grad.cpu() - gref[k]).abs().max().item() / gref[k].abs().max().item()
        assert err <= 0.03, (k, err)
    assert net.model.model3_1.UPNet[2].weight.grad is not None and net.model.model4_1.UPNet[2].weight.grad is None


@pytest.mark.parametrize("kind", ["l1", "l2", "cb"])
def test_fused_pixel_loss_matches_get_loss(golden_dir, kind):
    """bin_b200.loss.pixel_loss vs the reference's bin_model.get_loss (golden) and oracle autograd for the gradients."""
    from bin_b200.loss import pixel_loss
    g = {k: torch.from_numpy(v) for k, v in np.load(os.path.join(golden_dir, "get_loss.npz")).items()}
    outs = [t.clone().cuda().requires_grad_(True) for t in g["outs"]]
    gts = [t.clone().cuda() for t in g["gts"]]
    loss, ll = pixel_loss(outs, gts, kind)
    assert abs(loss.item() - g[kind].item()) <= 1e-5 * max(1.0, abs(g[kind].item()))
    assert (torch.stack(ll).cpu() - g[kind + "_list"]).abs().max().item() <= 1e-4 * max(1.0, g[kind + "_list"].abs().max().item())
    loss.backward()
    ro = [t.clone().requires_grad_(True) for t in g["outs"]]
    rl, _ = O.get_loss_6v2(ro, list(g["gts"]), kind)
    rg = torch.autograd.grad(rl, ro)
    for a, b in zip(outs, rg):
        assert (a.grad.cpu() - b).abs().max().item() <= 1e-5 * max(1.0, b.abs().max().item())
