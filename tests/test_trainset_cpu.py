"""CPU checks of the GPU training-set loader (bin_b200.trainset, bin_train_batch_u8): the NumPy restatement against the
reference's own BINDataset (tests/golden/trainset.npz), the C ABI's argument checks (no device needed), the header
struct layout, the constructors' validation, and the full reference run when BIN_REFERENCE names a checkout."""
import ctypes as C
import os
import random
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import trainset_oracle as TO


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "trainset.npz"))


_CLIPS = {}


def clip(folder):
    """(blurry, kept sharp, first, im_list) of a fixture clip, from its seed."""
    if folder not in _CLIPS:
        spec = {c[0]: c for c in TO.CLIPS}[folder]
        _, T, H, W, seed, omit = spec
        sharp, blurry, kept, first = TO.clip_arrays(T, H, W, seed)
        names = [TO.name(first + 8 * i) + ".png" for i in range(len(blurry))]
        _CLIPS[folder] = (sharp, blurry, kept, first, {n for n in names if n not in omit})
    return _CLIPS[folder]


def restate(listdir, h, w, seed, order):
    """The restated loader on the fixture clips in `listdir` order -> (keys, draws, sha256 per sample)."""
    rng = random.Random(seed)
    specs = [{"folder": f, "first": clip(f)[3], "nb": len(clip(f)[1]), "im_list": clip(f)[4]} for f in listdir]
    wins = TO.windows(specs, rng)
    draws, shas = [], []
    for i in order:
        ci, j, _ = wins[i]
        d = TO.draw(rng, h, w)
        s = TO.sample(clip(listdir[ci])[1], clip(listdir[ci])[2], j, d, h, w)
        draws.append(d)
        shas.append([TO.sha256(s[k]) for k in ("LQs", "GTenh", "GTinp")])
    return [k for _, _, k in wins], draws, shas


def test_fixture_clips_come_from_their_seeds(golden):
    for folder, *_ in TO.CLIPS:
        sharp, blurry = clip(folder)[:2]
        assert list(golden[f"clip_{folder}_sha256"]) == [TO.sha256(sharp), TO.sha256(blurry)]
    assert sorted(golden["listdir"]) == sorted(c[0] for c in TO.CLIPS)


@pytest.mark.parametrize("tag", sorted(TO.LQ_SIZES))
def test_restatement_reproduces_the_reference_loader(golden, tag):
    h, w, seed = (int(v) for v in golden[f"{tag}_meta"])
    assert (h, w) == TO.LQ_SIZES[tag]
    keys, draws, shas = restate(list(golden["listdir"]), h, w, seed, [int(i) for i in golden[f"{tag}_order"]])
    assert keys == list(golden[f"{tag}_keys"]) and len(keys) == 6       # 7 windows, one dropped by the im_list
    assert not any(k == "IMG_0030_00017" for k in keys)
    assert np.array_equal(np.array(draws), golden[f"{tag}_draws"])
    assert shas == golden[f"{tag}_sha256"].tolist()
    d = golden[f"{tag}_draws"]
    assert set(d[:, 0]) == {0, 1} and set(d[:, 3]) == {0, 1}          # both orders and both flips are pinned


def test_train_batch_abi_rejects_bad_arguments_without_a_device():
    """bin_train_batch_u8 checks every argument before its first CUDA call: each call here fails with BIN_ERR_ARG and
    its message (the pointers are fake and never dereferenced)."""
    from bin_b200 import _lib
    L = _lib.lib()
    buf = (C.c_ubyte * 64)()
    fake = C.addressof(buf)

    def table(n=1, H=352, W=640, top=0, left=0, flip=0, null_at=None):
        t = (_lib.TrainSample * max(n, 1))()
        for e in t:
            for f in range(_lib.BIN_TRAIN_FRAMES):
                e.src[f] = fake
            e.H, e.W, e.top, e.left, e.flip = H, W, top, left, flip
        if null_at is not None:
            t[null_at[0]].src[null_at[1]] = None
        return t

    cases = [  # (table, B, h, w, dst, dst_B, b0), error text
        ((None, 1, 8, 8, fake, 1, 0), "null table"),
        ((table(), 0, 8, 8, fake, 1, 0), "B must be 1..16"),
        ((table(17), 17, 8, 8, fake, 17, 0), "B must be 1..16"),
        ((table(), -1, 8, 8, fake, 1, 0), "B must be 1..16"),
        ((table(), 1, 0, 8, fake, 1, 0), "h and w must be >= 1"),
        ((table(), 1, 8, -3, fake, 1, 0), "h and w must be >= 1"),
        ((table(), 1, 8, 8, None, 1, 0), "null dst"),
        ((table(), 1, 8, 8, fake, 1, -1), "must lie inside dst_B"),
        ((table(2), 2, 8, 8, fake, 2, 1), "must lie inside dst_B"),
        ((table(), 1, 8, 8, fake, 0, 0), "must lie inside dst_B"),
        ((table(), 1, 1 << 20, 1 << 20, fake, 1 << 30, 0), "dst too large"),
        ((table(3, null_at=(2, 16)), 3, 8, 8, fake, 3, 0), "null frame pointer"),
        ((table(flip=2), 1, 8, 8, fake, 1, 0), "flip must be 0 or 1"),
        ((table(flip=-1), 1, 8, 8, fake, 1, 0), "flip must be 0 or 1"),
        ((table(H=0), 1, 8, 8, fake, 1, 0), "source H and W must be >= 1"),
        ((table(H=(1 << 31) - 1, W=(1 << 31) - 1), 1, 8, 8, fake, 1, 0), "source frame too large"),
        ((table(top=345), 1, 8, 8, fake, 1, 0), "crop outside its source frame"),
        ((table(left=633), 1, 8, 8, fake, 1, 0), "crop outside its source frame"),
        ((table(top=-1), 1, 8, 8, fake, 1, 0), "crop outside its source frame"),
        ((table(left=-1), 1, 8, 8, fake, 1, 0), "crop outside its source frame"),
        ((table(H=4, W=4), 1, 8, 8, fake, 1, 0), "crop outside its source frame"),
        ((table(top=(1 << 31) - 4), 1, 8, 8, fake, 1, 0), "crop outside its source frame"),
    ]
    for (tab, B, h, w, dst, dst_B, b0), text in cases:
        ptr = None if tab is None else C.cast(tab, C.POINTER(_lib.TrainSample))
        rc = L.bin_train_batch_u8(ptr, B, h, w, dst, dst_B, b0, None)
        err = L.bin_last_error().decode()
        assert rc == 1 and text in err and err.startswith("train_batch_u8:"), (B, h, w, dst_B, b0, rc, err)


def test_train_sample_struct_matches_the_header(tmp_path):
    """sizeof / offsetof of bin_train_sample_t as gcc sees include/bin_b200.h == the ctypes mirror, and 16 samples fit
    the 4 KB of kernel parameters with room for the rest."""
    from bin_b200 import _lib
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    fields = [f[0] for f in _lib.TrainSample._fields_]
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "bin_b200.h"', 'int main(void) {',
             '  printf("size %zu\\n", sizeof(bin_train_sample_t));',
             '  printf("max %d %d\\n", BIN_TRAIN_MAX_BATCH, BIN_TRAIN_FRAMES);']
    lines += [f'  printf("{f} %zu\\n", offsetof(bin_train_sample_t, {f}));' for f in fields]
    lines += ['  return 0;', '}']
    src = tmp_path / "probe.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "probe"
    subprocess.run(["gcc", "-I", os.path.join(root, "include"), str(src), "-o", str(exe)], check=True)
    got = {l.split(" ", 1)[0]: l.split(" ", 1)[1] for l in
           subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines()}
    assert int(got["size"]) == C.sizeof(_lib.TrainSample)
    assert got["max"] == f"{_lib.BIN_TRAIN_MAX_BATCH} {_lib.BIN_TRAIN_FRAMES}" == "16 17"
    for f in fields:
        assert int(got[f]) == getattr(_lib.TrainSample, f).offset, f
    assert _lib.BIN_TRAIN_MAX_BATCH * C.sizeof(_lib.TrainSample) + 64 < 4096


def _frames(n, H=352, W=640, dtype=torch.uint8):
    return torch.zeros((1, 1, 1, 1), dtype=dtype).expand(n, H, W, 3)       # no memory behind the shape


def test_device_clip_validation():
    from bin_b200 import BinB200Error
    from bin_b200.trainset import DeviceClip
    bad = [
        ((_frames(8, dtype=torch.float32), _frames(15)), "uint8"),
        ((np.zeros((8, 352, 640, 3), np.uint8), _frames(15)), "uint8"),
        ((_frames(8)[..., :2], _frames(15)), r"\(n,H,W,3\)"),
        ((_frames(8)[0], _frames(15)), r"\(n,H,W,3\)"),
        ((_frames(8), _frames(15, 360, 656)), "share H and W"),
        ((_frames(8, 351, 640), _frames(15, 351, 640)), "crops inside 352x640"),
        ((_frames(8, 352, 639), _frames(15, 352, 639)), "crops inside 352x640"),
        ((_frames(8), _frames(14)), "read 15 sharp frames, got 14"),
        ((_frames(8), _frames(15)), "CUDA"),                       # valid shapes: refused only for the device
        ((_frames(8, 360, 656), _frames(15, 360, 656)), "CUDA"),
    ]
    for (b, s), text in bad:
        with pytest.raises(BinB200Error, match=text):
            DeviceClip("c", b, s)
    with pytest.raises(BinB200Error, match="first_index"):
        DeviceClip("c", _frames(8), _frames(15), first_index=-1)
    with pytest.raises(BinB200Error, match="CUDA"):
        DeviceClip("c", _frames(3), _frames(1))                    # fewer than 6 blurry frames: no windows to feed
    with pytest.raises(BinB200Error, match="CUDA"):
        DeviceClip.from_sharp("c", _frames(72))


def test_dataset_and_op_validation_without_a_device():
    from bin_b200 import BinB200Error, ops
    from bin_b200.trainset import DeviceBINDataset
    for size in ((3, 353, 256), (3, 128, 641), (3, 0, 8), (3, 8, 0)):
        with pytest.raises(BinB200Error, match="must crop inside 352x640"):
            DeviceBINDataset([], lq_size=size)
    ds = DeviceBINDataset([], lq_size=(3, 352, 640))
    assert len(ds) == 0 and ds.keys == []
    with pytest.raises(BinB200Error, match="batch_size"):
        next(ds.batches([0], 0))
    with pytest.raises(BinB200Error, match="no samples"):
        ops.train_batch_u8([], 8, 8)
    with pytest.raises(BinB200Error, match="CUDA"):
        ops.train_batch_u8([([_frames(1)[0]] * 17, 0, 0, 0)], 8, 8)


def test_reference_loader_matches_the_restatement(tmp_path):
    """The unmodified data/BIN_dataset.py on a cv2-written tree gives the restatement's keys, draws and bytes (in the
    tree's own listdir order).  Needs a reference checkout named by BIN_REFERENCE; skipped without one."""
    ref = os.environ.get("BIN_REFERENCE", "")
    if not os.path.isfile(os.path.join(ref, "data", "BIN_dataset.py")):
        pytest.skip("set BIN_REFERENCE to a checkout of the reference (laomao0/BIN) to run this test")
    pytest.importorskip("cv2")
    saved = {k: sys.modules.pop(k) for k in list(sys.modules) if k == "data" or k.startswith("data.")}
    sys.path.insert(0, ref)
    try:
        from data.BIN_dataset import BINDataset
        TO.write_tree(str(tmp_path))
        listdir = os.listdir(tmp_path / "train_blur")
        for tag, (h, w) in TO.LQ_SIZES.items():
            opt = {"dataroot_GT": str(tmp_path), "dataroot_LQ": str(tmp_path), "data_type": "img",
                   "LQ_size": [3, h, w], "name": "train"}
            state = random.getstate()
            random.seed(11)
            ds = BINDataset(opt)
            order = [0, 5, 2, 2, 4]
            got = [ds[i] for i in order]
            random.setstate(state)
            keys, _, shas = restate(listdir, h, w, 11, order)
            assert [p[3] for p in ds.all_paths] == keys
            assert [s["key"] for s in got] == [keys[i] for i in order]
            assert [[TO.sha256(s[k].numpy()) for k in ("LQs", "GTenh", "GTinp")] for s in got] == shas
    finally:
        sys.path.remove(ref)
        for k in [k for k in sys.modules if k == "data" or k.startswith("data.")]:
            sys.modules.pop(k)
        sys.modules.update(saved)
