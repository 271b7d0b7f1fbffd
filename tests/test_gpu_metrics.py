"""GPU checks of bin_image_metrics_u8 and the drop-ins of bin_b200.metrics: against the reference's own utils/util.py
results (tests/golden/metrics.npz), against the fp64 oracle at test.py's frame size, analytic cases, bit
reproducibility (repeats, workspace reuse, side streams) and test.py's exact call pattern through the skimage shim."""
import math
import os

import numpy as np
import pytest
import torch

from oracle import metrics_oracle as M

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "metrics.npz"))


def _exact_sums(a, b):
    d = a.astype(np.int64) - b.astype(np.int64)
    return int(np.abs(d).sum()), int((d * d).sum())


def _pair(kind, shape, seed):
    rng = np.random.default_rng(seed)
    if kind == "noise":
        a = rng.integers(0, 256, size=shape, dtype=np.uint8)
        u = rng.integers(0, 256, size=shape, dtype=np.uint8)
        return a, np.round(0.5 * a + 0.5 * u).astype(np.uint8)
    from scipy.ndimage import gaussian_filter
    z = gaussian_filter(rng.standard_normal(shape), sigma=(4.0, 4.0) + (0.0,) * (len(shape) - 2))
    a = np.clip(np.round((z - z.min()) / (z.max() - z.min()) * 235 + 10), 0, 255).astype(np.uint8)
    b = np.clip(a.astype(np.int32) + rng.normal(0, 4, size=shape).round().astype(np.int32), 0, 255).astype(np.uint8)
    return a, b


def test_fixture_pairs_match_the_reference(golden):
    from bin_b200 import metrics
    for n in golden["names"]:
        a, b = golden[f"{n}_a"], golden[f"{n}_b"]
        mean_abs, mse, g, bx = metrics.image_metrics(torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda())
        s_abs, s_sq = _exact_sums(a, b)
        assert mean_abs == s_abs / a.size and mse == s_sq / a.size, n                       # exact sums
        ref = float(golden[f"{n}_ssim"])
        if min(a.shape[:2]) < 11:
            assert math.isnan(ref) and math.isnan(g) and math.isnan(metrics.calculate_ssim(a, b)), n
        else:
            assert abs(g - ref) <= 1e-10, (n, g, ref)
            assert abs(metrics.calculate_ssim(a, b) - ref) <= 1e-10, n
        assert abs(bx - M.ssim_box7(a, b)) <= 1e-10, n
        assert metrics.calculate_psnr(a, b) == float(golden[f"{n}_psnr"]), n                # bit for bit
        assert metrics.compare_psnr(a, b) == float(golden[f"{n}_psnr_sk"]), n


CASES = [("noise", (720, 1280, 3)), ("smooth", (720, 1280, 3)), ("smooth", (768, 1344, 3)), ("noise", (11, 11, 3)),
         ("noise", (7, 9, 3)), ("smooth", (37, 53, 3)), ("noise", (33, 70)), ("smooth", (95, 64)),
         ("smooth", (61, 47, 1)), ("noise", (7, 7, 1)), ("noise", (45, 33, 3))]


@pytest.mark.parametrize("kind,shape", CASES, ids=[f"{k}-{'x'.join(map(str, s))}" for k, s in CASES])
def test_against_the_oracle(kind, shape):
    """Both SSIMs within 1e-10 of the fp64 restatements, sums exact; the sizes cover partial last tiles in both
    directions, single-tile images, the 7-pixel minimum and the Gaussian's 11-pixel minimum."""
    from bin_b200 import metrics
    a, b = _pair(kind, shape, seed=CASES.index((kind, shape)))
    mean_abs, mse, g, bx = metrics.image_metrics(torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda())
    s_abs, s_sq = _exact_sums(a, b)
    assert mean_abs == s_abs / a.size and mse == s_sq / a.size
    if min(shape[:2]) < 11:
        assert math.isnan(g)
    else:
        assert abs(g - M.ssim_gauss11(a, b)) <= 1e-10, (g, M.ssim_gauss11(a, b))
    assert abs(bx - M.ssim_box7(a, b)) <= 1e-10, (bx, M.ssim_box7(a, b))


def test_identical_and_constant_images():
    from bin_b200 import metrics
    a, _ = _pair("noise", (75, 130, 3), 3)
    ta = torch.from_numpy(a).cuda()
    mean_abs, mse, g, bx = metrics.image_metrics(ta, ta.clone())
    assert mean_abs == 0 and mse == 0 and abs(g - 1) <= 1e-15 and abs(bx - 1) <= 1e-15
    assert metrics.calculate_psnr(a, a) == float("inf") and metrics.compare_psnr(a, a) == float("inf")
    for av, bv in ((0, 255), (10, 200), (128, 128), (255, 3)):
        x, y = np.full((20, 24, 3), av, np.uint8), np.full((20, 24, 3), bv, np.uint8)
        want = (2 * av * bv + M.C1) / (av * av + bv * bv + M.C1)
        _, _, g, bx = metrics.image_metrics(x, y)
        assert abs(g - want) <= 1e-12 and abs(bx - want) <= 1e-15, (av, bv, g, bx, want)


def _raw(a, b, stream=None):
    """One bin_image_metrics_u8 call -> the 4 result doubles as raw bits."""
    from bin_b200 import _lib
    from bin_b200.rdn import _workspace
    L = _lib.lib()
    h, w = a.shape[:2]
    c = 1 if a.dim() == 2 else a.shape[2]
    s = stream or torch.cuda.current_stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ws = _workspace(a.device, L.bin_image_metrics_workspace_bytes(h, w))
        out = torch.full((4,), float("nan"), dtype=torch.float64, device=a.device)
        _lib.check(L.bin_image_metrics_u8(a.data_ptr(), b.data_ptr(), h, w, c, out.data_ptr(), ws.data_ptr(), ws.numel(),
                                          s.cuda_stream))
    s.synchronize()
    return out.cpu().numpy().view(np.uint64).tolist()


def test_bit_reproducible_across_repeats_workspace_reuse_and_streams():
    a, b = (torch.from_numpy(x).cuda() for x in _pair("smooth", (720, 1280, 3), 11))
    a0, b0 = a.clone(), b.clone()
    first = _raw(a, b)
    assert [_raw(a, b) for _ in range(2)] == [first, first]
    big_a, big_b = (torch.from_numpy(x).cuda() for x in _pair("noise", (1080, 1920, 3), 12))
    _raw(big_a, big_b)                                                # a larger pair refills the shared workspace
    small_a, small_b = (torch.from_numpy(x).cuda() for x in _pair("noise", (40, 40, 3), 13))
    _raw(small_a, small_b)
    assert _raw(a, b) == first
    side = torch.cuda.Stream()
    assert _raw(a, b, side) == first
    assert torch.equal(a, a0) and torch.equal(b, b0)                  # inputs untouched


def test_test_py_call_pattern_through_the_shim(monkeypatch):
    """test.py:33-35 and :404-458: numpy uint8 RGB arrays made with img[:, :, [2, 1, 0]] (test.py:58-66), then
    compare_ssim(res, gt, multichannel=True) and compare_psnr(res, gt)."""
    import sys
    from bin_b200 import metrics
    for k in ("skimage", "skimage.measure"):       # sys.modules is restored afterwards: stubs the shim adds are removed
        monkeypatch.setitem(sys.modules, k, sys.modules.get(k))
        if sys.modules[k] is None:
            monkeypatch.delitem(sys.modules, k)
    metrics.install_skimage_measure()
    ns = {}
    exec("from skimage.measure import compare_ssim,compare_psnr\n"
         "def my_compare_ssim(img1,img2):\n"
         "    ssim = compare_ssim(img1, img2, multichannel=True)\n"
         "    return ssim\n", ns)
    res_bgr, gt_bgr = _pair("smooth", (720, 1280, 3), 21)
    res, gt = res_bgr[:, :, [2, 1, 0]], gt_bgr[:, :, [2, 1, 0]]
    psnr_tmp = ns["compare_psnr"](res, gt)
    ssim_tmp = ns["my_compare_ssim"](res, gt)
    assert isinstance(psnr_tmp, np.float64) and isinstance(ssim_tmp, np.float64)
    assert psnr_tmp == M.psnr_skimage(res, gt)
    assert abs(ssim_tmp - M.ssim_box7(res, gt)) <= 1e-10
    assert 0.5 < ssim_tmp < 1 and 20 < psnr_tmp < 60
    # the util path (use_default_ssim = 0, test.py:39-40)
    assert metrics.calculate_psnr(res, gt) == M.psnr(res, gt)
    assert abs(metrics.calculate_ssim(res, gt) - M.ssim_gauss11(res, gt)) <= 1e-10
