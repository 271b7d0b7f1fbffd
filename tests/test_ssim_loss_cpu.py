"""The 'cb+ssim' criterion's host side (DESIGN §4r): the fp64 SSIM oracle against the reference's own utils/util.py
(tests/golden/ssim_loss.npz, written by oracle/make_golden_ssim.py), the train yml keys, the unchanged print line of
the other criteria, and the refusal of images too small for the 11 x 11 window."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from bin_b200 import BinB200Error
from bin_b200 import train as T
from oracle import ssim_oracle as S

from test_train_driver_cpu import with_


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "ssim_loss.npz"))


def test_oracle_matches_the_reference_util(golden):
    names = list(golden["names"])
    assert len(names) == 13
    for n in names:
        a = torch.from_numpy(golden[f"{n}_a"]).double()[None]
        b = torch.from_numpy(golden[f"{n}_b"]).double()[None]
        got = S.ssim(a, b).item()                            # data range 1; the reference ran on x * 255
        for key in ("ssim", "calc"):
            assert abs(got - float(golden[f"{n}_{key}"])) <= 1e-12, (n, key, got)
    assert float(golden["identical_24x31_ssim"]) == 1.0
    assert (golden["wide_24x31_a"].min() < -0.2) and (golden["wide_24x31_a"].max() > 1.2)


def test_oracle_constant_images_have_the_closed_form():
    a, b = torch.full((1, 3, 11, 12), 0.25, dtype=torch.float64), torch.full((1, 3, 11, 12), 0.75, dtype=torch.float64)
    want = (2 * 0.25 * 0.75 + S.C1) / (0.25 ** 2 + 0.75 ** 2 + S.C1)
    assert S.ssim_map(a, b).shape == (1, 3, 1, 2)
    assert abs(S.ssim(a, b).item() - want) <= 1e-12


def test_options_accept_cb_ssim_with_its_weight():
    o = T.parse_options(with_(**{"train.pixel_criterion": "cb+ssim"}))
    assert (o.pixel_criterion, o.ssim_weight) == ("cb+ssim", 0.01)
    o = T.parse_options(with_(**{"train.pixel_criterion": "cb+ssim", "train.ssim_weight": 0.5}))
    assert o.ssim_weight == 0.5
    for crit in ("l1", "l2", "cb"):                          # read only with cb+ssim
        assert T.parse_options(with_(**{"train.pixel_criterion": crit})).ssim_weight is None
        assert T.parse_options(with_(**{"train.pixel_criterion": crit, "train.ssim_weight": None})).ssim_weight is None


def test_options_refuse_cb_ssim_without_its_weight():
    with pytest.raises(BinB200Error, match=r"train\.ssim_weight is missing"):
        T.parse_options(with_(**{"train.pixel_criterion": "cb+ssim", "train.ssim_weight": None}))
    with pytest.raises(BinB200Error, match=r"train\.pixel_criterion"):
        T.parse_options(with_(**{"train.pixel_criterion": "ssim"}))


def test_print_line_is_unchanged_for_the_other_criteria():
    avg = [0.001 * (i + 1) for i in range(15)]
    old = "<epoch:  3, iter:  12,345, lr:1.000e-04> " + \
        " ".join("{}: {:.4e}".format(k, v) for k, v in zip([str(i) for i in range(14)] + ["Al"], avg))
    assert T.train_message(3, 12345, 1e-4, avg, None) == old
    assert T.train_message(3, 12345, 1e-4, avg, None, None) == old
    assert T.train_message(3, 12345, 1e-4, avg, (2, 3.5)) == old + " skipped: 2 grad_norm: 3.5000e+00"
    assert T.train_message(3, 12345, 1e-4, avg, None, 0.00125) == old + " ssim_loss: 1.2500e-03"
    assert T.train_message(3, 12345, 1e-4, avg, (0, None), 0.5) == \
        old + " ssim_loss: 5.0000e-01 skipped: 0 grad_norm: n/a"


@pytest.mark.parametrize("h,w", [(10, 11), (11, 10), (5, 64), (64, 1)])
def test_sizes_below_11_are_refused(h, w):
    from bin_b200.loss import pixel_loss, ssim
    a, b = torch.zeros(2, 3, h, w), torch.zeros(2, 3, h, w)
    with pytest.raises(BinB200Error, match="at least 11"):
        ssim(a, b)
    with pytest.raises(BinB200Error, match="at least 11"):
        pixel_loss([a] * 14, [b] * 14, "cb+ssim", ssim_weight=0.01)
    from bin_b200._lib import lib
    assert lib().bin_ssim_loss_scratch_bytes(1, 6, h, w) == 0 and lib().bin_ssim_loss_maps_bytes(1, 6, h, w) == 0
    fake = (C.c_void_p * 1)(16)                               # refused before any pointer is read
    out = C.c_void_p(16)
    assert lib().bin_ssim_loss_fwd(fake, fake, 1, 6, h, w, out, None, 0, None, 0, None) != 0
    assert "at least 11" in lib().bin_last_error().decode()
    assert lib().bin_ssim_loss_bwd(fake, fake, out, fake, None, 1, 6, h, w, out, None) != 0
    assert "at least 11" in lib().bin_last_error().decode()


def test_cb_ssim_needs_its_weight_and_shapes():
    from bin_b200.loss import pixel_loss, ssim
    a = torch.zeros(1, 3, 16, 16)
    with pytest.raises(BinB200Error, match="ssim_weight"):
        pixel_loss([a] * 14, [a] * 14, "cb+ssim")
    with pytest.raises(BinB200Error, match="shapes differ"):
        ssim(a, torch.zeros(1, 3, 16, 17))
    with pytest.raises(BinB200Error, match=r"\(B, C, H, W\)"):
        ssim(a[0], a[0])
    with pytest.raises(BinB200Error, match="CUDA tensors only"):
        ssim(a, a)


def test_scratch_and_maps_bytes():
    from bin_b200._lib import lib
    # 17 terms of a (2, 3, 128, 256) batch: 6 planes of 118 x 246 positions, 4 x 8 tiles of 32 x 32
    assert lib().bin_ssim_loss_scratch_bytes(17, 6, 128, 256) == 17 * 6 * 4 * 8 * 4
    assert lib().bin_ssim_loss_maps_bytes(17, 6, 128, 256) == 17 * 4 * 6 * 118 * 246 * 4
    assert lib().bin_ssim_loss_scratch_bytes(21, 6, 128, 256) == 0
