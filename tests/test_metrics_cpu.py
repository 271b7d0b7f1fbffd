"""CPU checks of the evaluation metrics (bin_b200.metrics): the fp64 oracle against the reference's own
utils/util.py results, the analytic cases that pin the skimage restatement, the C ABI's argument checks (no device
needed) and the skimage.measure shim."""
import ctypes as C
import importlib.util
import os
import sys
import types

import numpy as np
import pytest

from oracle import metrics_oracle as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "metrics.npz"))


def test_oracle_matches_the_reference_util(golden):
    """ssim_gauss11 / psnr against calculate_ssim / calculate_psnr of the unmodified utils/util.py."""
    assert np.array_equal(golden["gauss11"], M.GAUSS11)
    names = list(golden["names"])
    assert len(names) == 10
    spread = []
    for n in names:
        a, b = golden[f"{n}_a"], golden[f"{n}_b"]
        ref = float(golden[f"{n}_ssim"])
        got = M.ssim_gauss11(a, b)
        if min(a.shape[:2]) < 11:
            assert np.isnan(ref) and np.isnan(got), n
        else:
            assert abs(got - ref) <= 1e-12, (n, got, ref)
            spread.append(ref)
        assert M.psnr(a, b) == float(golden[f"{n}_psnr"]), n                  # bit for bit
        assert M.psnr_skimage(a, b) == float(golden[f"{n}_psnr_sk"]), n
    assert min(spread) < 0.35 and max(spread) > 0.98                          # low- and high-SSIM pairs


@pytest.mark.parametrize("fn", [M.ssim_gauss11, M.ssim_box7])
def test_oracle_analytic_cases(fn):
    """Identical images give 1; constant images a, b give (2ab+C1)/(a^2+b^2+C1) (every variance is 0)."""
    rng = np.random.default_rng(5)
    for shape in ((23, 31, 3), (19, 12), (15, 16, 1)):
        x = rng.integers(0, 256, size=shape, dtype=np.uint8)
        assert abs(fn(x, x) - 1.0) <= 1e-15
    for av in (0, 1, 10, 100, 128, 200, 255):
        for bv in (0, 3, 50, 128, 255):
            a, b = np.full((13, 17, 3), av, np.uint8), np.full((13, 17, 3), bv, np.uint8)
            want = (2 * av * bv + M.C1) / (av * av + bv * bv + M.C1)
            assert abs(fn(a, b) - want) <= 1e-15, (av, bv)


def test_image_metrics_rejects_bad_arguments_without_a_device():
    """bin_image_metrics_u8 checks every argument before its first CUDA call: each call here fails with BIN_ERR_ARG
    and its message (the pointers are fake and never dereferenced)."""
    from bin_b200 import _lib
    L = _lib.lib()
    assert L.bin_image_metrics_workspace_bytes(720, 1280) == 23 * 40 * 32
    assert L.bin_image_metrics_workspace_bytes(7, 7) == 32 and L.bin_image_metrics_workspace_bytes(6, 100) == 0
    buf = (C.c_double * 64)()
    p = C.addressof(buf)
    ws = L.bin_image_metrics_workspace_bytes(64, 64)
    cases = [  # (a, b, h, w, c, out4, workspace, workspace_bytes), error text
        ((None, p, 64, 64, 3, p, p, ws), "null argument"),
        ((p, None, 64, 64, 3, p, p, ws), "null argument"),
        ((p, p, 64, 64, 3, None, p, ws), "null argument"),
        ((p, p, 64, 64, 3, p, None, ws), "null argument"),
        ((p, p, 64, 64, 2, p, p, ws), "c must be 1 or 3"),
        ((p, p, 64, 64, 0, p, p, ws), "c must be 1 or 3"),
        ((p, p, 6, 64, 3, p, p, ws), "at least 7"),
        ((p, p, 64, 6, 1, p, p, ws), "at least 7"),
        ((p, p, 70000, 64, 1, p, p, ws), "too large"),
        ((p, p, 30000, 30000, 3, p, p, ws), "too large"),
        ((p, p, 64, 64, 3, p + 4, p, ws), "aligned"),
        ((p, p, 64, 64, 3, p, p, ws - 1), "workspace too small"),
        ((p, p, 65, 64, 3, p, p, ws), "workspace too small"),
    ]
    for args, text in cases:
        rc = L.bin_image_metrics_u8(*args, None)
        err = L.bin_last_error().decode()
        assert rc == 1 and text in err and err.startswith("image_metrics:"), (args[2:5], rc, err)


@pytest.fixture
def clean_skimage(monkeypatch):
    """Run with no skimage modules registered, and restore sys.modules afterwards."""
    for k in [k for k in sys.modules if k == "skimage" or k.startswith("skimage.")]:
        monkeypatch.delitem(sys.modules, k)
    saved = dict(sys.modules)
    yield
    for k in [k for k in sys.modules if k == "skimage" or k.startswith("skimage.")]:
        if k not in saved:
            del sys.modules[k]


def _test_py_import():
    ns = {}
    exec("from skimage.measure import compare_ssim,compare_psnr", ns)        # test.py:33 verbatim
    return ns["compare_ssim"], ns["compare_psnr"]


def test_shim_installs_without_skimage(clean_skimage):
    from bin_b200 import metrics
    if importlib.util.find_spec("skimage") is not None:
        pytest.skip("a real scikit-image is installed")
    with pytest.raises(ImportError):
        _test_py_import()
    m1 = metrics.install_skimage_measure()
    m2 = metrics.install_skimage_measure()                                      # idempotent
    assert m1 is m2 is sys.modules["skimage.measure"] and sys.modules["skimage"].measure is m1
    assert _test_py_import() == (metrics.compare_ssim, metrics.compare_psnr)


def test_shim_extends_an_existing_skimage(clean_skimage):
    """An importable skimage.measure gets the two attributes and keeps everything else."""
    from bin_b200 import metrics
    sk, measure = types.ModuleType("skimage"), types.ModuleType("skimage.measure")
    sk.__path__, sk.measure = [], measure
    sentinel = object()
    measure.label = sentinel
    measure.compare_mse = sentinel
    sys.modules["skimage"], sys.modules["skimage.measure"] = sk, measure
    before = dict(vars(measure))
    assert metrics.install_skimage_measure() is measure
    metrics.install_skimage_measure()
    assert sys.modules["skimage.measure"] is measure and sys.modules["skimage"] is sk
    assert measure.label is sentinel and measure.compare_mse is sentinel
    assert set(vars(measure)) - set(before) == {"compare_ssim", "compare_psnr"}
    assert _test_py_import() == (metrics.compare_ssim, metrics.compare_psnr)


def test_metric_functions_without_a_device_raise():
    import torch
    from bin_b200 import BinB200Error, metrics
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    a = np.zeros((16, 16, 3), np.uint8)
    for fn in (metrics.calculate_psnr, metrics.calculate_ssim, metrics.compare_psnr, metrics.image_metrics):
        with pytest.raises(BinB200Error):
            fn(a, a)
    with pytest.raises(BinB200Error):
        metrics.compare_ssim(a, a, multichannel=True)
    with pytest.raises(BinB200Error):
        metrics.image_metrics(torch.zeros((16, 16, 3), dtype=torch.uint8), torch.zeros((16, 16, 3), dtype=torch.uint8))


def test_unsupported_options_and_inputs_raise():
    """Only the defaults test.py uses are implemented; every other option value names itself.  Checked before any
    device work, so this runs anywhere."""
    from bin_b200 import BinB200Error, metrics
    a = np.zeros((16, 16, 3), np.uint8)
    g = a[:, :, 0]
    bad = [({"win_size": 11}, "win_size"), ({"gradient": True}, "gradient"), ({"data_range": 1.0}, "data_range"),
           ({"gaussian_weights": True}, "gaussian_weights"), ({"full": True}, "full"), ({"K1": 0.02}, "K1"),
           ({"K2": 0.05}, "K2"), ({"sigma": 2.0}, "sigma"), ({"use_sample_covariance": False}, "use_sample_covariance"),
           ({"mode": "constant"}, "mode")]
    for kw, name in bad:
        with pytest.raises(BinB200Error, match=name):
            metrics.compare_ssim(a, a, multichannel=True, **kw)
    with pytest.raises(BinB200Error, match="multichannel"):
        metrics.compare_ssim(a, a)                       # skimage would run a 3-D 7x7x7 window here
    with pytest.raises(BinB200Error, match="multichannel"):
        metrics.compare_ssim(g, g, multichannel=True)
    with pytest.raises(BinB200Error, match="data_range"):
        metrics.compare_psnr(a, a, data_range=1.0)
    f = a.astype(np.float32)
    for fn in (metrics.calculate_psnr, metrics.calculate_ssim, metrics.compare_psnr, metrics.image_metrics):
        with pytest.raises(BinB200Error, match="uint8"):
            fn(f, f)
    with pytest.raises(BinB200Error, match="uint8"):
        metrics.compare_ssim(f, f, multichannel=True)
    with pytest.raises(BinB200Error, match=r"\(h, w, 3\)"):
        metrics.image_metrics(np.zeros((9, 9, 2), np.uint8), np.zeros((9, 9, 2), np.uint8))
    # the reference's ValueErrors (utils/util.py:239-252, skimage _assert_compatible)
    for fn in (metrics.calculate_psnr, metrics.calculate_ssim, metrics.compare_psnr):
        with pytest.raises(ValueError, match="Input images must have the same dimensions."):
            fn(a, a[:8])
    with pytest.raises(ValueError, match="Input images must have the same dimensions."):
        metrics.compare_ssim(a, a[:8], multichannel=True)
    with pytest.raises(ValueError, match="Wrong input image dimensions."):
        metrics.calculate_ssim(a[None], a[None])
