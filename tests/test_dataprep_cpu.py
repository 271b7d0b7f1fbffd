"""CPU checks of the dataset builder (bin_b200.dataprep.build_dataset, python -m bin_b200.dataprep): the script's
arguments and defaults, the ffmpeg command against the argv the reference script gave the stub ffmpeg
(tests/golden/blur_tree.npz, oracle/make_golden_blur_tree.py), the skipped extraction and copy, every refusal, and the
window, chunk and name arithmetic against oracle.bin_oracle.blur_average and the fixture's lists."""
import json
import os

import numpy as np
import pytest

from bin_b200 import BinB200Error, dataprep as D
from oracle import bin_oracle as O
from oracle import make_golden_blur_tree as G


@pytest.fixture(scope="module")
def golden(golden_dir):
    d = np.load(os.path.join(golden_dir, "blur_tree.npz"))
    return {run: json.loads(str(d[run])) for run in G.RUNS}


def write_frames(folder, T, h=4, w=6, seed=0, names=None):
    import cv2
    os.makedirs(folder, exist_ok=True)
    frames = np.random.default_rng(seed).integers(0, 256, size=(T, h, w, 3), dtype=np.uint8)
    for k, f in enumerate(frames):
        assert cv2.imwrite(os.path.join(folder, names[k] if names else D.frame_name(k)), f)
    return frames


def write_list(path, videos):
    with open(path, "w") as fh:
        fh.write("\n".join(videos))
    return path


def nothing_of(root, split, stem):
    return not any(os.path.exists(os.path.join(root, *p)) for p in
                   ((split + "_blur", stem), (split, stem), (split + "_list", stem + "_im_list.txt")))


# ----------------------------------------------------------------------------- arguments
def test_parse_args_has_the_scripts_defaults():
    a = D.parse_args(["--dataset_folder", "out"])
    assert (a.dataset, a.img_width, a.img_height, a.window_size, a.enable_train) == ("adobe240fps_blur", 256, 128, 7, 0)
    assert a.ffmpeg_dir is None and a.videos_folder is None and a.dataset_folder == "out"
    assert a.test_list == "./test_list.txt" and a.train_list is None and a.decode_threads == 8
    a = D.parse_args(["--ffmpeg_dir", "f", "--dataset", "youtube240fps_blur", "--videos_folder", "v", "--dataset_folder",
                      "d", "--img_width", "640", "--img_height", "352", "--window_size", "11", "--enable_train", "1",
                      "--test_list", "t.txt", "--train_list", "l.txt", "--decode_threads", "3"])
    assert (a.ffmpeg_dir, a.dataset, a.videos_folder, a.img_width, a.img_height, a.window_size, a.enable_train,
            a.test_list, a.train_list, a.decode_threads) == ("f", "youtube240fps_blur", "v", 640, 352, 11, 1, "t.txt",
                                                             "l.txt", 3)
    with pytest.raises(SystemExit):
        D.parse_args([])                                        # --dataset_folder is required, as in the script


def test_train_list_defaults_to_the_scripts_path(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    write_list("test_list.txt", [])
    with pytest.raises(BinB200Error, match="adobe240fps/train_list.txt"):
        D.build_dataset(str(tmp_path / "d"), enable_train=1)
    with pytest.raises(BinB200Error, match="youtube240fps/train_list.txt"):
        D.build_dataset(str(tmp_path / "d"), enable_train=1, dataset="youtube240fps_blur")


# ----------------------------------------------------------------------------- extraction and copy
@pytest.mark.parametrize("run", list(G.RUNS))
def test_ffmpeg_command_matches_the_fixture(golden, tmp_path, monkeypatch, run):
    opt = G.RUNS[run]
    bin_dir = G.write_stub(str(tmp_path / "bin"))
    log = str(tmp_path / "argv.jsonl")
    monkeypatch.setenv(G.LOG_ENV, log)
    data, videos = str(tmp_path / "data"), str(tmp_path / "videos")
    root = os.path.join(data, "full_sharp")
    for v in G.TEST + G.TRAIN:
        assert D.extract_frames(v, videos, root, bin_dir, opt["img_width"], opt["img_height"])
        stem = os.path.splitext(v)[0]
        assert D.frame_count(os.path.join(root, stem)) == G.VIDEOS[v][0]
    with open(log) as fh:
        argvs = [json.loads(line) for line in fh]
    for key, path in (("dataset_folder", data), ("videos_folder", videos), ("ffmpeg_dir", bin_dir)):
        argvs = [[x.replace(path, "{" + key + "}") for x in a] for a in argvs]
    assert argvs == golden[run]["argv"]
    full = sorted(os.path.relpath(os.path.join(d, n), data) for d, _, ns in os.walk(root) for n in ns)
    assert full == [f for f in golden[run]["files"] if f.startswith("full_sharp" + os.sep)]


def test_extraction_and_copy_are_skipped_when_the_folders_exist(tmp_path, monkeypatch):
    bin_dir = G.write_stub(str(tmp_path / "bin"))
    log = str(tmp_path / "argv.jsonl")
    monkeypatch.setenv(G.LOG_ENV, log)
    data = str(tmp_path / "data")
    os.makedirs(os.path.join(data, "full_sharp", "clip_a"))
    assert not D.extract_frames("clip_a.mp4", "videos", os.path.join(data, "full_sharp"), bin_dir, 640, 352)
    assert not os.path.exists(log)                              # ffmpeg never ran
    # a clip of 20 frames has no window (floor(20/8) - 2 = 0): the whole run needs no device
    write_frames(os.path.join(data, "full_sharp", "short"), 20)
    write_frames(os.path.join(data, "full_sharp", "kept"), 20, seed=1)
    write_frames(os.path.join(data, "test", "kept"), 2, seed=2)             # already there: left as it is
    lst = write_list(str(tmp_path / "t.txt"), ["short.mp4", "kept.mov"])
    done = D.build_dataset(data, test_list=lst, ffmpeg_dir=bin_dir, videos_folder="videos")
    assert not os.path.exists(log)
    assert [(v.stem, v.frames, v.blurry, v.extracted, v.copied) for v in done] == \
        [("short", 20, 0, False, True), ("kept", 20, 0, False, False)]
    assert sorted(os.listdir(os.path.join(data, "test", "short"))) == [D.frame_name(k) for k in range(20)]
    assert sorted(os.listdir(os.path.join(data, "test", "kept"))) == [D.frame_name(k) for k in range(2)]
    for stem in ("short", "kept"):
        assert not os.path.exists(os.path.join(data, "test_blur", stem))   # the script makes it per blurry frame
        with open(os.path.join(data, "test_list", stem + "_im_list.txt"), "rb") as fh:
            assert fh.read() == b""
    assert sorted(os.listdir(data)) == sorted(["full_sharp", "train", "test", "train_list", "test_list", "train_blur",
                                               "test_blur"])


def test_empty_lines_of_a_list_are_skipped(tmp_path):
    data = str(tmp_path / "data")
    write_frames(os.path.join(data, "full_sharp", "short"), 20)
    lst = str(tmp_path / "t.txt")
    with open(lst, "w") as fh:
        fh.write("\nshort.mp4\n\n")
    assert [v.stem for v in D.build_dataset(data, test_list=lst)] == ["short"]


# ----------------------------------------------------------------------------- refusals
def test_refuses_a_gap_in_the_names(tmp_path):
    data = str(tmp_path / "data")
    write_frames(os.path.join(data, "full_sharp", "v"), 40, names=[D.frame_name(k) for k in range(41) if k != 17])
    with pytest.raises(BinB200Error, match="found 00019.png where 00018.png belongs"):
        D.build_dataset(data, test_list=write_list(str(tmp_path / "t.txt"), ["v.mp4"]))
    assert nothing_of(data, "test", "v")


def test_refuses_names_that_do_not_start_at_00001(tmp_path):
    data = str(tmp_path / "data")
    write_frames(os.path.join(data, "full_sharp", "v"), 30, names=[D.frame_name(k + 1) for k in range(30)])
    with pytest.raises(BinB200Error, match="00001.png"):
        D.build_dataset(data, test_list=write_list(str(tmp_path / "t.txt"), ["v.mp4"]))
    os.makedirs(os.path.join(data, "full_sharp", "empty"))
    with pytest.raises(BinB200Error, match="holds no frames"):
        D.build_dataset(data, test_list=write_list(str(tmp_path / "t.txt"), ["empty.mp4"]))


def test_refuses_a_missing_full_sharp_folder_without_ffmpeg(tmp_path):
    data = str(tmp_path / "data")
    write_frames(os.path.join(data, "full_sharp", "short"), 20)
    lst = write_list(str(tmp_path / "t.txt"), ["short.mp4", "absent.mp4"])
    with pytest.raises(BinB200Error, match=r"full_sharp/absent does not exist"):
        D.build_dataset(data, test_list=lst)
    assert not os.path.exists(os.path.join(data, "test", "short"))         # checked before any video is processed
    with pytest.raises(BinB200Error, match="videos_folder"):
        D.build_dataset(data, test_list=lst, ffmpeg_dir=str(tmp_path))


def test_refuses_a_failed_ffmpeg(tmp_path):
    bin_dir = str(tmp_path / "bin")
    os.makedirs(bin_dir)
    with open(os.path.join(bin_dir, "ffmpeg"), "w") as fh:
        fh.write("#!/bin/sh\nexit 3\n")
    os.chmod(os.path.join(bin_dir, "ffmpeg"), 0o755)
    data = str(tmp_path / "data")
    lst = write_list(str(tmp_path / "t.txt"), ["v.mp4"])
    with pytest.raises(BinB200Error, match=r"ffmpeg failed on v.mp4 \(3\)"):
        D.build_dataset(data, test_list=lst, ffmpeg_dir=bin_dir, videos_folder=str(tmp_path))
    assert not os.path.exists(os.path.join(data, "full_sharp", "v"))       # the next run extracts again
    assert nothing_of(data, "test", "v")
    with pytest.raises(BinB200Error, match="ffmpeg failed"):                # no ffmpeg there at all
        D.build_dataset(data, test_list=lst, ffmpeg_dir=str(tmp_path / "none"), videos_folder=str(tmp_path))


def test_refuses_the_custom_dataset(tmp_path):
    lst = write_list(str(tmp_path / "t.txt"), [])
    with pytest.raises(BinB200Error, match="two of its five arguments"):
        D.build_dataset(str(tmp_path / "d"), test_list=lst, dataset="custom")
    assert not os.path.exists(str(tmp_path / "d"))


def test_refuses_a_missing_list(tmp_path):
    with pytest.raises(BinB200Error, match="nolist.txt does not exist"):
        D.build_dataset(str(tmp_path / "d"), test_list=str(tmp_path / "nolist.txt"))
    lst = write_list(str(tmp_path / "t.txt"), [])
    with pytest.raises(BinB200Error, match="notrain.txt does not exist"):
        D.build_dataset(str(tmp_path / "d"), test_list=lst, train_list=str(tmp_path / "notrain.txt"), enable_train=1)
    D.build_dataset(str(tmp_path / "d"), test_list=lst, train_list=str(tmp_path / "notrain.txt"))   # not read


@pytest.mark.parametrize("T,ws", [(40, 17), (47, 31), (64, 35), (40, 300)])
def test_refuses_a_window_outside_the_frames(tmp_path, T, ws):
    data = str(tmp_path / "data")
    write_frames(os.path.join(data, "full_sharp", "v"), T)
    with pytest.raises(BinB200Error, match="window_size"):
        D.build_dataset(data, test_list=write_list(str(tmp_path / "t.txt"), ["v.mp4"]), window_size=ws)
    assert nothing_of(data, "test", "v")


def test_window_size_limits():
    assert D.window_mids(40, 15) == [16, 24, 32]                # frames 9..39: the last frame is read
    with pytest.raises(BinB200Error):
        D.window_mids(40, 17)                                   # frame 40 of 0..39
    assert D.window_mids(47, 29) == [16, 24, 32]                # T = 8k + 7: 14 frames past the last middle
    with pytest.raises(BinB200Error):
        D.window_mids(47, 31)


def test_refuses_a_frame_that_is_not_8_bit_3_channel(tmp_path):
    import cv2
    good = str(tmp_path / "good.png")
    assert cv2.imwrite(good, np.zeros((4, 5, 3), np.uint8))
    assert D.read_frame(good).shape == (4, 5, 3)
    for name, img in (("gray.png", np.zeros((4, 5), np.uint8)), ("rgba.png", np.zeros((4, 5, 4), np.uint8)),
                      ("deep.png", np.zeros((4, 5, 3), np.uint16))):
        path = str(tmp_path / name)
        assert cv2.imwrite(path, img)
        with pytest.raises(BinB200Error, match=name):
            D.read_frame(path)
    with pytest.raises(BinB200Error, match="cannot read"):
        D.read_frame(str(tmp_path / "missing.png"))


# ----------------------------------------------------------------------------- windows, chunks and names
@pytest.mark.parametrize("ws", [1, 3, 7, 8, 11, 13, 15])
@pytest.mark.parametrize("per_chunk", [1, 3, 16])
def test_chunks_give_the_oracles_blur(ws, per_chunk):
    for T in (24, 31, 40, 41, 64, 97, 150):
        frames = np.random.default_rng(T + ws).integers(0, 256, size=(T, 2, 3, 3), dtype=np.uint8)
        mids = D.window_mids(T, ws)
        want = O.blur_average(frames, window_size=ws)
        assert len(mids) == len(want) == D.window_count(T)
        parts = []
        r = int((ws - 1) / 2)
        for chunk, lo, hi in D.chunks(mids, ws, per_chunk):
            assert 1 <= len(chunk) <= per_chunk and lo == chunk[0] - r and hi == chunk[-1] + r
            parts.append(O.blur_average(frames[lo:hi + 1], window_size=ws, first_mid=chunk[0] - lo, nwin=len(chunk)))
        assert np.array_equal(np.concatenate(parts), want)
        # script :113-128: window w's file is its middle frame, 0-based 16 + 8w, named from 1
        assert [D.frame_name(m) for m in mids] == ["{}".format(16 + 8 * w + 1).zfill(5) + ".png"
                                                   for w in range(len(want))]


@pytest.mark.parametrize("run", list(G.RUNS))
def test_names_match_the_fixture(golden, run):
    g = golden[run]
    ws = G.RUNS[run]["window_size"]
    for split, videos in (("test", G.TEST), ("train", G.TRAIN)):
        for v in videos:
            stem = os.path.splitext(v)[0]
            names = [D.frame_name(m) for m in D.window_mids(G.VIDEOS[v][0], ws)]
            assert g["lists"][os.path.join(split + "_list", stem + "_im_list.txt")] == "\n".join(names)
            blur = os.path.join(split + "_blur", stem) + os.sep
            assert sorted(f[len(blur):] for f in g["files"] if f.startswith(blur)) == names
            copy = os.path.join(split, stem) + os.sep
            assert sorted(f[len(copy):] for f in g["files"] if f.startswith(copy)) == \
                [D.frame_name(k) for k in range(G.VIDEOS[v][0])]
    assert len(g["argv"]) == len(G.TEST) + len(G.TRAIN)
