"""The dataset builder on the GPU: build_dataset with the stub ffmpeg against the tree the reference's own script wrote
(tests/golden/blur_tree.npz: the paths, the list texts, the ffmpeg argv and the decoded pixels of every blurry frame
and sharp copy), the same files whatever the chunk size, DeviceBINDataset.from_tree on the built train split against
DeviceClip.from_sharp of the same frames, a second run over a finished tree, and the command line followed by
evaluate_testset on the test split it wrote."""
import json
import os
import random
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import arch_oracle as A
from oracle import make_golden_blur_tree as G

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build(tmp, run, monkeypatch, data=None, ffmpeg=True):
    """build_dataset with RUNS[run]'s options over TEST and TRAIN, extracting with the stub ffmpeg.
    -> (dataset folder, the VideoDone list, describe() of the tree)."""
    from bin_b200 import dataprep as D
    os.makedirs(tmp, exist_ok=True)
    G.write_lists(tmp)
    bin_dir = G.write_stub(os.path.join(tmp, "bin"))
    log = os.path.join(tmp, "argv.jsonl")
    if os.path.exists(log):
        os.remove(log)
    monkeypatch.setenv(G.LOG_ENV, log)
    data = data or os.path.join(tmp, "data")
    videos = os.path.join(tmp, "videos")
    opt = G.RUNS[run]
    done = D.build_dataset(data, test_list=os.path.join(tmp, "test_list.txt"),
                           train_list=os.path.join(tmp, "adobe240fps", "train_list.txt"), videos_folder=videos,
                           ffmpeg_dir=bin_dir if ffmpeg else None, img_width=opt["img_width"],
                           img_height=opt["img_height"], window_size=opt["window_size"], enable_train=1,
                           decode_threads=4)
    return data, done, G.describe(data, log, {"dataset_folder": data, "videos_folder": videos, "ffmpeg_dir": bin_dir})


def file_bytes(root, tops=("test_blur", "train_blur", "test_list", "train_list", "test", "train")):
    out = {}
    for top in tops:
        for d, _, names in os.walk(os.path.join(root, top)):
            for n in names:
                with open(os.path.join(d, n), "rb") as fh:
                    out[os.path.relpath(os.path.join(d, n), root)] = fh.read()
    return out


@pytest.fixture(scope="module")
def golden(golden_dir):
    d = np.load(os.path.join(golden_dir, "blur_tree.npz"))
    return {run: json.loads(str(d[run])) for run in G.RUNS}


@pytest.fixture(scope="module")
def built(tmp_path_factory):
    mp = pytest.MonkeyPatch()
    try:
        return {run: build(str(tmp_path_factory.mktemp(run)), run, mp) for run in G.RUNS}
    finally:
        mp.undo()


@pytest.mark.parametrize("run", list(G.RUNS))
def test_tree_matches_the_reference_script(golden, built, run):
    _, done, got = built[run]
    want = golden[run]
    assert got["files"] == want["files"]
    assert got["dirs"] == want["dirs"]
    assert got["lists"] == want["lists"]
    assert got["argv"] == want["argv"]
    assert got["sha"] == want["sha"]
    assert [(v.split, v.stem, v.frames, v.extracted, v.copied) for v in done] == \
        [(s, os.path.splitext(v)[0], G.VIDEOS[v][0], True, True) for s, vs in (("test", G.TEST), ("train", G.TRAIN))
         for v in vs]


@pytest.mark.parametrize("per_chunk", [1, 3])
@pytest.mark.parametrize("run", list(G.RUNS))
def test_chunk_size_does_not_change_the_files(built, tmp_path, monkeypatch, run, per_chunk):
    from bin_b200 import dataprep as D
    src = built[run][0]
    data = str(tmp_path / "data")
    shutil.copytree(os.path.join(src, "full_sharp"), os.path.join(data, "full_sharp"))
    monkeypatch.setattr(D, "CHUNK_WINDOWS", per_chunk)
    build(str(tmp_path), run, monkeypatch, data=data, ffmpeg=False)
    assert file_bytes(data) == file_bytes(src)


def test_from_tree_equals_from_sharp(built):
    """The built train split read as the reference's loader reads it, against the clip synthesised from the same
    sharp frames on the device: the same keys and the same batch bytes for one seed."""
    import cv2
    from bin_b200.trainset import DeviceBINDataset, DeviceClip
    data = built["ws11"][0]
    stem = os.path.splitext(G.TRAIN[0])[0]
    folder = os.path.join(data, "full_sharp", stem)
    sharp = np.stack([cv2.imread(os.path.join(folder, n)) for n in sorted(os.listdir(folder))])
    with open(os.path.join(data, "train_list", stem + "_im_list.txt")) as fh:
        im_list = fh.read().split("\n")
    random.seed(31)
    a = DeviceBINDataset.from_tree(data, "train")
    got_a = [a.batch(range(k, k + 2)) for k in range(0, len(a) - 1, 2)]
    random.seed(31)
    b = DeviceBINDataset([DeviceClip.from_sharp(stem, torch.from_numpy(sharp).cuda(), window_size=11,
                                                im_list=im_list)])
    got_b = [b.batch(range(k, k + 2)) for k in range(0, len(b) - 1, 2)]
    assert a.keys == b.keys and len(a.keys) == 5
    for x, y in zip(got_a, got_b):
        assert x["key"] == y["key"]
        for k in ("LQs", "GTenh", "GTinp"):
            assert torch.equal(x[k], y[k]), k


def test_second_run_skips_extraction_and_copy(built, tmp_path, monkeypatch):
    src = built["ws7"][0]
    data = str(tmp_path / "data")
    shutil.copytree(src, data)
    before = file_bytes(data, ("test", "train"))
    _, done, got = build(str(tmp_path), "ws7", monkeypatch, data=data)
    assert got["argv"] == []
    assert not any(v.extracted or v.copied for v in done)
    assert file_bytes(data, ("test", "train")) == before
    assert got["sha"] == built["ws7"][2]["sha"]


def test_refuses_a_bad_frame_mid_video(tmp_path):
    import cv2
    from bin_b200 import BinB200Error, dataprep as D
    g = np.random.default_rng(3)
    for name, bad in (("gray", np.zeros((24, 40), np.uint8)), ("size", np.zeros((24, 41, 3), np.uint8))):
        data = str(tmp_path / name)
        folder = os.path.join(data, "full_sharp", "v")
        os.makedirs(folder)
        for k in range(64):
            img = bad if k == 45 else g.integers(0, 256, size=(24, 40, 3), dtype=np.uint8)
            assert cv2.imwrite(os.path.join(folder, D.frame_name(k)), img)
        lst = str(tmp_path / "list.txt")
        with open(lst, "w") as fh:
            fh.write("v.mp4")
        with pytest.raises(BinB200Error, match="00046.png"):
            D.build_dataset(data, test_list=lst, window_size=11)
        assert not os.path.exists(os.path.join(data, "test", "v"))


def test_command_line_then_evaluate(tmp_path):
    """python -m bin_b200.dataprep on frames already under full_sharp, then evaluate_testset on the test split."""
    import cv2
    from bin_b200 import dataprep as D, rdn
    from bin_b200.evaluate import evaluate_testset
    data = str(tmp_path / "D")
    g = np.random.default_rng(8)
    for stem, T in (("v1", 41), ("v2", 48)):
        folder = os.path.join(data, "full_sharp", stem)
        os.makedirs(folder)
        base = g.integers(0, 256, size=(10, 14, 3)).astype(np.float32)
        for k in range(T):
            img = cv2.resize(base + g.normal(0, 8, size=base.shape).astype(np.float32), (48, 32))
            assert cv2.imwrite(os.path.join(folder, D.frame_name(k)), np.clip(img, 0, 255).astype(np.uint8))
    lists = {}
    for split, videos in (("test", ["v1.mp4", "v2.mov"]), ("train", ["v2.mov"])):
        lists[split] = str(tmp_path / f"{split}.txt")
        with open(lists[split], "w") as fh:
            fh.write("\n".join(videos))
    r = subprocess.run([sys.executable, "-m", "bin_b200.dataprep", "--dataset_folder", data, "--test_list",
                        lists["test"], "--train_list", lists["train"], "--enable_train", "1", "--window_size", "11"],
                       cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.splitlines() == ["test v1: 41 frames -> 3 blurry frames", "test v2: 48 frames -> 4 blurry frames",
                                     "train v2: 48 frames -> 4 blurry frames"]
    assert sorted(os.listdir(os.path.join(data, "test_blur", "v2"))) == ["00017.png", "00025.png", "00033.png",
                                                                         "00041.png"]
    net = rdn.bin_stage4_lstm()
    net.model = rdn.RDN_residual_interp_5_input(lstm=True, GO=64, D=6)
    net.load_state_dict(A.synth_state_dict(0, 64, 6), strict=True)
    net = net.cuda().eval()
    out = str(tmp_path / "eval")
    summary = evaluate_testset(net, os.path.join(data, "test_blur"), os.path.join(data, "test"), out, "bin",
                               decode_threads=2)
    gen = os.path.join(out, "60fps_test_results", "bin")
    assert os.path.isfile(summary)
    # test.py writes 2n - 2 images for n blurry frames: n - 1 interpolated, n - 2 second deblurred and the first one
    assert len(os.listdir(os.path.join(gen, "v1"))) == 2 * 3 - 2 and len(os.listdir(os.path.join(gen, "v2"))) == 2 * 4 - 2
