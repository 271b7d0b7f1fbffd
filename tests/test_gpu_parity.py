"""Parity of the sm_90a path (through the C ABI / the nn.Module mirror) against
(a) the golden fixtures produced by the unmodified reference and (b) the fp32 CPU oracle.

Tolerance (north_star / BASELINE.md §4): fp16 storage + fp32 accumulate -> max-abs <= 1e-3 on the
network outputs; the ConvLSTM and layout kernels are fp32 -> <= 1e-5; PSNR within 0.01 dB."""
import os

import numpy as np
import pytest
import torch

from oracle import bin_oracle as O

pytestmark = pytest.mark.gpu
TOL_FP16 = 1e-3
TOL_FP32 = 1e-5


def _load(golden_dir, name):
    return {k: torch.from_numpy(v) for k, v in np.load(os.path.join(golden_dir, name)).items()}


@pytest.fixture(scope="module")
def net():
    from bin_b200 import rdn
    m = rdn.bin_stage4_lstm()
    m.load_state_dict(O.synth_state_dict(0), strict=True)
    return m.cuda().eval()


@pytest.fixture(scope="module")
def sd():
    return O.synth_state_dict(0)


def test_device_is_b200():
    from bin_b200 import _lib
    _lib.check(_lib.lib().bin_check_device())


def test_pixel_reshuffle_bit_exact(golden_dir):
    from bin_b200 import rdn
    g = _load(golden_dir, "pixel_reshuffle.npz")
    got = rdn.pixel_reshuffle(g["x"].cuda(), 2).cpu()
    assert torch.equal(got, g["out"])        # small integers: exact in fp16


def test_convlstm_golden(golden_dir, net):
    g = _load(golden_dir, "convlstm.npz")
    cell = net.clstm_7_prime_prime
    with torch.no_grad():
        h, (c, h2) = cell(g["x"].cuda(), None)
        assert (h.cpu() - g["h_none"]).abs().max() <= TOL_FP32 and (c.cpu() - g["c_none"]).abs().max() <= TOL_FP32
        h, (c, _) = cell(g["x"].cuda(), [g["c0"].cuda(), g["h0"].cuda()])
        assert (h.cpu() - g["h_state"]).abs().max() <= TOL_FP32 and (c.cpu() - g["c_state"]).abs().max() <= TOL_FP32


def test_rdb_golden(golden_dir, net):
    g = _load(golden_dir, "rdb.npz")
    blk = net.model.model2_1.RDBs[3]
    with torch.no_grad():
        y = blk(g["x"].cuda()).cpu()
    ref = g["out"]
    # inputs ~N(0,1): compare relative to the activation scale (fp16 storage of |x| up to ~5)
    assert (y - ref).abs().max().item() <= 4e-3 * ref.abs().max().item()


@pytest.mark.parametrize("B,H,W", [(1, 4, 30), (2, 6, 34), (1, 10, 64), (3, 5, 31), (1, 2, 2), (2, 48, 100), (1, 129, 61)])
def test_rdb_shapes_vs_oracle(net, sd, B, H, W):
    """The fused conv3 + LFF tail (rdb_tail.cu: 4-row x 30-column tiles, pipelined over tiles) on ragged sizes:
    partial tiles in x and y, single-tile launches, several tiles per CTA (129 x 61 = 99 tiles... x B)."""
    from bin_b200._lib import check, lib
    prefix = "model.model3_1.RDBs.7"
    x = torch.randn((B, 96, H, W), generator=torch.Generator().manual_seed(H * 131 + W))
    ref = O.rdb(x, sd, prefix)
    blob = net.model.model3_1.packed_blob()                 # bin_rdb_fwd = the backbone's own RDB walker (run_rdb)
    xc, y = x.cuda(), torch.empty((B, 96, H, W), device="cuda")
    ws = torch.empty(B * 40 * H * W * 16 + 1024, dtype=torch.uint8, device="cuda")
    check(lib().bin_rdb_fwd(blob.data_ptr(), 5, 7, xc.data_ptr(), y.data_ptr(), B, H, W, ws.data_ptr(), ws.numel(),
                            torch.cuda.current_stream().cuda_stream))
    y = y.cpu()
    assert torch.isfinite(y).all()
    assert (y - ref).abs().max().item() <= 4e-3 * ref.abs().max().item()

@pytest.mark.parametrize("B,H,W,sub", [(2, 9, 37, (0, 0, 0, 0)), (3, 16, 64, (1, 2, 4, 7)), (1, 4, 30, (0, 1, 0, 4)), (1, 70, 45, (0, 0, 3, 0)),
                                       (4, 120, 200, (0, 0, 0, 0)),      # 840 tiles: 5-6 per CTA, both tile streams, 3 LFF accumulators
                                       (1, 148, 90, (0, 0, 0, 0))])      # 111 tiles... one per CTA on most, none on the rest
def test_rdb_tail_bit_identical_to_layerwise(B, H, W, sub):
    """bin_rdb_tail_fwd == conv3 (x-stacked kernel) followed by the LFF kernel, bit for bit (same accumulation order),
    on full tensors and on batch / row sub-ranges (rows outside the range must stay untouched)."""
    from bin_b200 import ops
    gen = torch.Generator(device="cuda").manual_seed(B * 1000 + H * 10 + W)
    rnd = lambda *sh: torch.randn(*sh, device="cuda", generator=gen)
    x, g = rnd(B, 12, H, W, 8).half(), rnd(B, 16, H, W, 8).half()
    w3, wl = rnd(32, 192, 3, 3) / 1728 ** 0.5, rnd(96, 224, 1, 1) / 224 ** 0.5
    b3, bl = ops.pad_bias(rnd(32) * 0.1, 32), ops.pad_bias(rnd(96) * 0.1, 96)
    p3, pl = ops.pack_conv_weight(w3, 32, 192), ops.pack_conv_weight(wl, 96, 224)
    g_ref = g.clone()
    sentinel = torch.full((B, 12, H, W, 8), 7.0, device="cuda").half()
    out_ref, out = sentinel.clone(), sentinel.clone()
    s4 = None if sub == (0, 0, 0, 0) else sub
    ops.conv_fwd(x, p3, b3, 3, 32, in0_planes=12, in1=g_ref, in1_planes=12, relu=True, out=g_ref, out_plane0=12, sub=s4)
    ops.conv_fwd(x, pl, bl, 1, 96, in0_planes=12, in1=g_ref, in1_planes=16, out=out_ref, res=x, sub=s4)
    ops.rdb_tail_fwd(x, g, p3, b3, pl, bl, out, sub=sub)
    torch.cuda.synchronize()
    assert torch.equal(g[:, :12], g_ref[:, :12])                    # inputs untouched, g3 never written
    assert torch.equal(out, out_ref)
    b0, nb, y0, ny = sub
    rows = torch.zeros(B, H, dtype=torch.bool)
    rows[b0:(b0 + nb) if nb else B, y0:(y0 + ny) if ny else H] = True
    written = (out != sentinel).any(dim=(1, 3, 4)).cpu()
    assert not (written & ~rows).any()

@pytest.mark.parametrize("name,n", [("model1_1", 2), ("model2_1", 3), ("model3_1", 5), ("model4_1", 5)])
def test_backbone_golden(golden_dir, net, name, n):
    g = _load(golden_dir, f"backbone_{name}.npz")
    fr = [f.cuda() for f in O.synth_frames(n, 2, 20, 36, seed=100 + n)]
    with torch.no_grad():
        y = getattr(net.model, name)(*fr).cpu()
    assert (y - g["out"]).abs().max().item() <= TOL_FP16


def test_pyramid_golden(golden_dir, net):
    g = _load(golden_dir, "pyramid.npz")
    fr = [f.cuda() for f in O.synth_frames(5, 1, 16, 24, seed=77)]
    prev = [(t * 2 - 1).cuda() for t in O.synth_frames(6, 1, 16, 24, seed=78)]
    with torch.no_grad():
        for tag, p in (("none", [None] * 6), ("prev", prev)):
            outs = net.model(*fr, p)
            for k, o in enumerate(outs):
                assert (o.cpu() - g[f"{tag}{k}"]).abs().max().item() <= TOL_FP16, (tag, k)


@pytest.mark.parametrize("tag", ["window_a", "window_b"])
def test_window_golden(golden_dir, net, tag):
    g = _load(golden_dir, tag + ".npz")
    B, H, W, smooth, seed, _ = [int(v) for v in g["meta"]]
    fr = [f.cuda() for f in O.synth_frames(6, B, H, W, seed=seed, smooth=bool(smooth))]
    with torch.no_grad():
        outs = net(*fr)
    assert len(outs) == 14
    worst = max((o.cpu() - g[f"out{k}"]).abs().max().item() for k, o in enumerate(outs))
    assert worst <= TOL_FP16, worst


@pytest.mark.parametrize("B,H,W", [(1, 64, 64), (1, 46, 122), (2, 32, 66)])
def test_window_vs_oracle_and_psnr(net, sd, B, H, W):
    """Edge shapes (tile remainders in both axes, batch > 1) against the CPU oracle + PSNR delta."""
    fr = O.synth_frames(6, B, H, W, seed=1234, smooth=True)
    gt = O.synth_frames(14, B, H, W, seed=4321, smooth=True)
    ref = O.window_forward(fr, sd)
    with torch.no_grad():
        outs = net(*[f.cuda() for f in fr])
    for k in range(14):
        got = outs[k].cpu()
        assert (got - ref[k]).abs().max().item() <= TOL_FP16, k
        p_ref = O.psnr_u8(O.tensor2img_u8(ref[k]), O.tensor2img_u8(gt[k]))
        p_got = O.psnr_u8(O.tensor2img_u8(got), O.tensor2img_u8(gt[k]))
        assert abs(p_ref - p_got) <= 0.01, (k, p_ref, p_got)


def test_pyramid3_config2a(net, sd):
    fr = O.synth_frames(4, 1, 40, 72, seed=5)
    ref = O.pyramid3_4frames(fr, sd)
    with torch.no_grad():
        outs = net.forward_pyramid3(*[f.cuda() for f in fr])
    for k in range(6):
        assert (outs[k].cpu() - ref[k]).abs().max().item() <= TOL_FP16, k


def test_config1_one_scale_on_four_frames(net, sd):
    """BASELINE config 1: stage 1 only on the 3 adjacent pairs of a 4 x (1,3,64,64) window (SURVEY 8d row 1)."""
    fr = O.synth_frames(4, 1, 64, 64, seed=1234)
    m1 = O.sub_sd(sd, "model.model1_1")
    with torch.no_grad():
        for a in range(3):
            ref = O.backbone((fr[a], fr[a + 1]), m1)
            got = net.model.model1_1(fr[a].cuda(), fr[a + 1].cuda()).cpu()
            assert (got - ref).abs().max().item() <= TOL_FP16, a


def test_dataparallel_wrapper_like_bin_model(net):
    """bin_model.py:42 wraps netG in nn.DataParallel; with one visible device the wrapper calls the module directly."""
    dp = torch.nn.DataParallel(net, device_ids=[0])
    fr = [f.cuda() for f in O.synth_frames(6, 1, 32, 32, seed=2)]
    with torch.no_grad():
        a, b = dp(*fr), net(*fr)
    assert len(a) == 14 and all(torch.equal(x, y) for x, y in zip(a, b))
    assert dp.module is net


def test_replica_packs_leave_the_masters_cache_alone(net):
    """An nn.DataParallel replica (bin_model.py:42) starts from a shallow copy of the master's __dict__, packed-weight
    caches included, and holds other weight tensors: packing those must cache on the replica only, so the master's next
    call still returns its own blob, in both precisions."""
    bb = net.model.model3_1
    blobs = [bb.packed_blob(prec) for prec in (0, 1)]
    # what replicate() does to one module tree, as in test_module_cpu's weight-walk test: copy every module, drop
    # _parameters, set plain tensor attributes
    mods = list(bb.modules())
    copies = {id(m): m._replicate_for_data_parallel() for m in mods}
    for m in mods:
        r = copies[id(m)]
        for key, child in m._modules.items():
            setattr(r, key, copies[id(child)])
        for key, p in m._parameters.items():
            setattr(r, key, p.detach() * 2.0)
    rep = copies[id(bb)]
    for prec, blob in zip((0, 1), blobs):
        rblob = rep.packed_blob(prec)
        assert rblob is not blob and rep.packed_blob(prec) is rblob
        assert bb.packed_blob(prec) is blob


def test_inputs_not_mutated_and_outputs_fresh(net):
    fr = [f.cuda() for f in O.synth_frames(6, 1, 32, 32, seed=2)]
    keep = [f.clone() for f in fr]
    with torch.no_grad():
        o1 = net(*fr)
        o2 = net(*fr)
    assert all(torch.equal(a, b) for a, b in zip(fr, keep))
    assert all(torch.equal(a, b) for a, b in zip(o1, o2))            # deterministic
    assert len({o.data_ptr() for o in o1 + o2}) == 28


def test_weight_update_invalidates_pack(net, sd):
    fr = [f.cuda() for f in O.synth_frames(6, 1, 32, 32, seed=2)]
    with torch.no_grad():
        a = net(*fr)[13].clone()
        w = net.model.model4_1.UPNet[2].bias
        keep = w.clone()
        w.add_(0.25)
        b = net(*fr)[13].clone()
        w.copy_(keep)
        c = net(*fr)[13].clone()
    assert (b - a - 0.25).abs().max().item() <= 1e-5 and torch.equal(a, c)


def test_full_size_properties(net):
    """720p: no oracle run (minutes on CPU) -- size-independent properties instead: finite outputs,
    translation of all inputs by a constant c translates outputs by c only through the mean path is
    NOT a property of this net, so check batch consistency: window(B=2 stack) == two B=1 windows."""
    H, W = 720, 1280
    fa = [f.cuda() for f in O.synth_frames(6, 1, H, W, seed=11, smooth=True)]
    fb = [f.cuda() for f in O.synth_frames(6, 1, H, W, seed=12, smooth=True)]
    with torch.no_grad():
        oa = net(*fa)
        ob = net(*fb)
        oab = net(*[torch.cat((a, b), 0) for a, b in zip(fa, fb)])
    for k in range(14):
        assert torch.isfinite(oab[k]).all()
        assert torch.equal(oab[k][0:1], oa[k]) and torch.equal(oab[k][1:2], ob[k]), k


# ------------------------------------------------------------------ fp32-accurate mode (north_star: 1e-5 max-abs)
TOL_FP32_MODE = 1e-5


@pytest.fixture(scope="module")
def net32():
    from bin_b200 import rdn
    m = rdn.bin_stage4_lstm()
    m.load_state_dict(O.synth_state_dict(0), strict=True)
    return rdn.set_precision(m.cuda().eval(), "fp32")


@pytest.mark.parametrize("name,n", [("model1_1", 2), ("model2_1", 3), ("model3_1", 5)])
def test_fp32_mode_backbone_golden(golden_dir, net32, name, n):
    g = _load(golden_dir, f"backbone_{name}.npz")
    fr = [f.cuda() for f in O.synth_frames(n, 2, 20, 36, seed=100 + n)]
    with torch.no_grad():
        y = getattr(net32.model, name)(*fr).cpu()
    assert (y - g["out"]).abs().max().item() <= TOL_FP32_MODE


@pytest.mark.parametrize("tag", ["window_a", "window_b"])
def test_fp32_mode_window_golden(golden_dir, net32, tag):
    g = _load(golden_dir, tag + ".npz")
    B, H, W, smooth, seed, _ = [int(v) for v in g["meta"]]
    fr = [f.cuda() for f in O.synth_frames(6, B, H, W, seed=seed, smooth=bool(smooth))]
    with torch.no_grad():
        outs = net32(*fr)
    worst = max((o.cpu() - g[f"out{k}"]).abs().max().item() for k, o in enumerate(outs))
    assert worst <= TOL_FP32_MODE, worst


def test_fp32_mode_window_vs_oracle(net32, sd):
    fr = O.synth_frames(6, 1, 46, 122, seed=1234, smooth=True)
    ref = O.window_forward(fr, sd)
    with torch.no_grad():
        outs = net32(*[f.cuda() for f in fr])
    worst = max((o.cpu() - r).abs().max().item() for o, r in zip(outs, ref))
    assert worst <= TOL_FP32_MODE, worst

