"""GPU checks of the training-set loader (bin_b200.trainset, bin_train_batch_u8): batches equal the NumPy restatement
(torch.equal) and the SHA-256 of the reference's own samples (tests/golden/trainset.npz) with the same keys and draws;
from_tree on a cv2-written tree; unmutated clips; the views of one buffer; and a training step fed by ds.batch equal to
one fed by the host batch."""
import os
import random

import numpy as np
import pytest
import torch

from oracle import bin_oracle as O
from oracle import trainset_oracle as TO

pytestmark = pytest.mark.gpu

ENH, INP = slice(6, 12), slice(12, 17)
# bin_model.get_info(mode=1) for nframes == 6 (bin_model.py:529-534): I(2k+1) = GTenh[:, k], I(2k+2) = GTinp[:, k]
GT_ORDER = ["I2", "I4", "I6", "I8", "I3", "I5", "I7", "I4", "I6", "I5", "I10", "I9", "I8", "I7"]


class Recording(random.Random):
    """random.Random that records what randint / choice return (the loader's four draws per sample)."""

    def __init__(self, seed):
        super().__init__(seed)
        self.drawn = []

    def randint(self, a, b):
        v = super().randint(a, b)
        self.drawn.append(v)
        return v

    def choice(self, seq):
        v = super().choice(seq)
        self.drawn.append(v)
        return v


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "trainset.npz"))


@pytest.fixture(scope="module")
def host():
    """folder -> (all sharp frames, blurry, kept sharp, first, im_list) on the host, from the fixture's seeds."""
    out = {}
    for folder, T, H, W, seed, omit in TO.CLIPS:
        sharp, blurry, kept, first = TO.clip_arrays(T, H, W, seed)
        names = [TO.name(first + 8 * i) + ".png" for i in range(len(blurry))]
        out[folder] = (sharp, blurry, kept, first, [n for n in names if n not in omit])
    return out


@pytest.fixture(scope="module")
def clips(golden, host):
    """DeviceClips in the fixture's listdir order, built from the sharp frames with DeviceClip.from_sharp."""
    from bin_b200.trainset import DeviceClip
    out = []
    for folder in golden["listdir"]:
        c = DeviceClip.from_sharp(str(folder), torch.from_numpy(host[str(folder)][0]).cuda(), im_list=host[str(folder)][4])
        assert torch.equal(c.blurry.cpu(), torch.from_numpy(host[str(folder)][1]))
        assert torch.equal(c.sharp.cpu(), torch.from_numpy(host[str(folder)][2]))
        out.append(c)
    return out


def restated(host, listdir, wins, i, d, h, w):
    ci, j = wins[i]
    _, blurry, kept, _, _ = host[str(listdir[ci])]
    s = TO.sample(blurry, kept, j, d, h, w)
    return np.concatenate([s["LQs"], s["GTenh"], s["GTinp"]])


def check_batch(b, golden, tag, host, wins, draws, n, h, w):
    """b: the batch of the first n fixture samples of `tag` -> equal to the restatement and to the fixture hashes."""
    assert b["LQs"].shape == (n, 6, 3, h, w) and b["GTenh"].shape == (n, 6, 3, h, w) and b["GTinp"].shape == (n, 5, 3, h, w)
    order = [int(i) for i in golden[f"{tag}_order"][:n]]
    assert b["key"] == [str(golden[f"{tag}_keys"][i]) for i in order]
    got = torch.cat([b["LQs"], b["GTenh"], b["GTinp"]], 1).cpu()
    for k, i in enumerate(order):
        ref = restated(host, golden["listdir"], wins, i, draws[k], h, w)
        assert torch.equal(got[k], torch.from_numpy(ref)), (tag, n, k)
        shas = [TO.sha256(got[k, 0:6].numpy()), TO.sha256(got[k, ENH].numpy()), TO.sha256(got[k, INP].numpy())]
        assert shas == golden[f"{tag}_sha256"][k].tolist(), (tag, n, k)


@pytest.mark.parametrize("B", [1, 3, 16, 17])
@pytest.mark.parametrize("tag", sorted(TO.LQ_SIZES))
def test_batch_matches_reference_fixture_and_restatement(golden, host, clips, tag, B):
    """Crops 128x256, 127x255 and 352x640 (the whole range: the 360x656 clip contributes its top-left only), clips of
    two sizes in one batch, both flips and orders; B = 17 takes two launches."""
    from bin_b200.trainset import DeviceBINDataset
    h, w, seed = (int(v) for v in golden[f"{tag}_meta"])
    rng = Recording(seed)
    ds = DeviceBINDataset(clips, lq_size=(3, h, w), rng=rng)
    assert ds.keys == list(golden[f"{tag}_keys"]) and len(ds) == 6
    wins = [(ci, j) for ci, c in enumerate(clips) for j, _ in c.windows()]
    random.Random(seed).shuffle(wins)
    b = ds.batch([int(i) for i in golden[f"{tag}_order"][:B]])
    torch.cuda.synchronize()
    draws = np.array(rng.drawn).reshape(B, 4)
    assert np.array_equal(draws, golden[f"{tag}_draws"][:B])
    check_batch(b, golden, tag, host, wins, draws, B, h, w)
    if B == 17:
        assert {d[0] for d in draws} == {0, 1} and {d[3] for d in draws} == {0, 1}
        sizes = {tuple(clips[wins[int(i)][0]].blurry.shape[1:3]) for i in golden[f"{tag}_order"][:B]}
        assert sizes == {(352, 640), (360, 656)}


@pytest.mark.parametrize("h,w", [(1, 1), (2, 640), (352, 1), (64, 96)])
def test_other_crops_match_the_restatement(host, clips, golden, h, w):
    from bin_b200.trainset import DeviceBINDataset
    rng = Recording(31 + h)
    ds = DeviceBINDataset(clips, lq_size=(3, h, w), rng=rng)
    wins = [(ci, j) for ci, c in enumerate(clips) for j, _ in c.windows()]
    random.Random(31 + h).shuffle(wins)
    order = [5, 0, 3, 3, 1, 2, 4, 4, 0, 5, 2, 1]
    b = ds.batch(order)
    draws = np.array(rng.drawn).reshape(len(order), 4)
    got = torch.cat([b["LQs"], b["GTenh"], b["GTinp"]], 1).cpu()
    for k, i in enumerate(order):
        assert torch.equal(got[k], torch.from_numpy(restated(host, golden["listdir"], wins, i, draws[k], h, w))), k
    assert b["key"] == [ds.keys[i] for i in order]


def test_getitem_batches_and_views(golden, clips):
    """ds[i] is __getitem__; batches() drops the last partial batch; the three tensors are views of one buffer whose
    per-frame slices LQs[:, k] are contiguous; the clips are never written."""
    from bin_b200.trainset import DeviceBINDataset
    before = [(c.blurry.clone(), c.sharp.clone()) for c in clips]
    ds = DeviceBINDataset(clips, lq_size=(3, 128, 256), rng=random.Random(int(golden["a_meta"][2])))
    s = ds[int(golden["a_order"][0])]
    assert s["LQs"].shape == (6, 3, 128, 256) and s["GTinp"].shape == (5, 3, 128, 256)
    assert s["key"] == str(golden["a_keys"][int(golden["a_order"][0])])
    assert TO.sha256(s["GTenh"].cpu().numpy()) == str(golden["a_sha256"][0][1])
    got = list(ds.batches(iter(range(7)), 3))
    assert len(got) == 2 and [b["key"] for b in got] == [ds.keys[0:3], ds.keys[3:6]]
    b = got[1]
    base = b["LQs"].data_ptr()
    plane = 3 * 3 * 128 * 256 * 4
    assert b["GTenh"].data_ptr() == base + 6 * plane and b["GTinp"].data_ptr() == base + 12 * plane
    assert len({t.untyped_storage().data_ptr() for t in (b["LQs"], b["GTenh"], b["GTinp"])}) == 1
    for t, n in ((b["LQs"], 6), (b["GTenh"], 6), (b["GTinp"], 5)):
        assert all(t[:, k].is_contiguous() for k in range(n))
        assert t[:, 0].to("cuda").data_ptr() == t[:, 0].data_ptr()          # feed_data's .to(device) copies nothing
    torch.cuda.synchronize()
    for c, (bl, sh) in zip(clips, before):
        assert torch.equal(c.blurry, bl) and torch.equal(c.sharp, sh)


def test_from_tree_equals_the_fixture(tmp_path, golden):
    pytest.importorskip("cv2")
    from bin_b200.trainset import DeviceBINDataset
    TO.write_tree(str(tmp_path))
    h, w, seed = (int(v) for v in golden["a_meta"])
    ds = DeviceBINDataset.from_tree(str(tmp_path), folders=[str(f) for f in golden["listdir"]], lq_size=(3, h, w),
                                    rng=random.Random(seed))
    assert ds.keys == list(golden["a_keys"])
    b = ds.batch([int(i) for i in golden["a_order"][:17]])
    got = torch.cat([b["LQs"], b["GTenh"], b["GTinp"]], 1).cpu()
    for k in range(17):
        shas = [TO.sha256(got[k, 0:6].numpy()), TO.sha256(got[k, ENH].numpy()), TO.sha256(got[k, INP].numpy())]
        assert shas == golden["a_sha256"][k].tolist(), k
    dflt = DeviceBINDataset.from_tree(str(tmp_path), rng=random.Random(seed))
    assert [c.name for c in dflt.clips] == os.listdir(tmp_path / "train_blur")
    omitted = [c for c in ds.clips if c.name == "IMG_0030"][0]
    assert int(omitted.blurry[0].sum()) == 0 and int(omitted.blurry[1].sum()) > 0   # window 0 dropped: file 17 unread


def test_refusals_on_the_device():
    from bin_b200 import BinB200Error, ops
    from bin_b200.trainset import DeviceClip
    z = torch.zeros((8, 352, 640, 3), dtype=torch.uint8, device="cuda")
    with pytest.raises(BinB200Error, match="read 15 sharp frames"):
        DeviceClip("c", z, z)
    with pytest.raises(BinB200Error, match="uint8"):
        DeviceClip("c", z.float(), z)
    f = torch.zeros((360, 656, 3), dtype=torch.uint8, device="cuda")
    with pytest.raises(BinB200Error, match="contiguous uint8"):
        ops.train_batch_u8([([f[:, :640]] * 17, 0, 0, 0)], 8, 8)
    with pytest.raises(BinB200Error, match="crop outside"):
        ops.train_batch_u8([([f] * 17, 300, 0, 0)], 64, 64)
    with pytest.raises(BinB200Error, match="flip must be 0 or 1"):
        ops.train_batch_u8([([f] * 17, 0, 0, 2)], 64, 64)


def _step(net, frames, gts):
    from bin_b200.loss import pixel_loss
    net.zero_grad(set_to_none=True)
    outs = net(*frames)
    loss, _ = pixel_loss(outs, gts, "l1")
    loss.backward()
    torch.cuda.synchronize()
    return [o.detach().clone() for o in outs], loss.item(), [p.grad.clone() for p in net.parameters()]


def _inputs(b):
    """feed_data (bin_model.py:147-202) + get_info(mode=1): the six frames and the 14 targets."""
    I = {f"I{2 * k + 1}": b["GTenh"][:, k] for k in range(6)}
    I.update({f"I{2 * k + 2}": b["GTinp"][:, k] for k in range(5)})
    return [b["LQs"][:, k] for k in range(6)], [I[n] for n in GT_ORDER]


def test_training_step_fed_by_the_device_batch(host, clips, golden):
    """A training step fed by ds.batch equals one fed by the restated host batch uploaded with .cuda(): the 14
    forward outputs bit for bit, the loss and every gradient within 1e-6 (the loss reduction adds with float atomics)."""
    from bin_b200 import rdn
    from bin_b200.trainset import DeviceBINDataset
    net = rdn.bin_stage4_lstm()
    net.load_state_dict(O.synth_state_dict(0), strict=True)
    net = net.cuda().train()
    rng = Recording(5)
    ds = DeviceBINDataset(clips, lq_size=(3, 128, 256), rng=rng)
    order = [3, 0]
    dev_b = ds.batch(order)
    wins = [(ci, j) for ci, c in enumerate(clips) for j, _ in c.windows()]
    random.Random(5).shuffle(wins)
    draws = np.array(rng.drawn).reshape(2, 4)
    hostbuf = np.stack([restated(host, golden["listdir"], wins, i, draws[k], 128, 256) for k, i in enumerate(order)])
    t = torch.from_numpy(hostbuf)
    host_b = {"LQs": t[:, 0:6], "GTenh": t[:, ENH], "GTinp": t[:, INP]}
    host_b = {k: v.contiguous().cuda() for k, v in host_b.items()}           # default_collate + .to(device)
    outs_a, loss_a, grads_a = _step(net, *_inputs(dev_b))
    outs_b, loss_b, grads_b = _step(net, *_inputs(host_b))
    assert all(torch.equal(a, b) for a, b in zip(outs_a, outs_b))
    assert abs(loss_a - loss_b) <= 1e-6 * abs(loss_b) and loss_b > 0
    assert len(grads_a) == 540
    for ga, gb in zip(grads_a, grads_b):
        assert (ga - gb).abs().max().item() <= 1e-6 * gb.abs().max().item()
