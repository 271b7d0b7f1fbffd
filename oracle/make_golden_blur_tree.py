"""Generate tests/golden/blur_tree.npz by EXECUTING THE REFERENCE'S OWN dataset script (CPU; needs the reference
checkout, and PIL or cv2):

    python oracle/make_golden_blur_tree.py /path/to/BIN

data_scripts/adobe240fps/create_dataset_blur_N_frames_average.py runs unmodified in a subprocess, once per entry of
RUNS, with the working directory holding its two video lists (TEST, TRAIN) and:

  * shims in sys.modules for the SciPy functions it imports, which SciPy 1.2 removed: scipy.ndimage.imread and
    scipy.misc.imsave backed by PIL (what those functions wrapped), or by cv2 with a channel swap if PIL is absent;
  * --ffmpeg_dir pointing at a stub `ffmpeg` (write_stub) that records its argv and writes the seeded frames
    (trainset_oracle.synth_clip) of the video it is given, VIDEOS[name] = (frame count, seed), at the size of its
    scale=W:H argument.

The fixture keeps no frames.  Per run: every file and directory written under --dataset_folder (relative paths), the
text of each _im_list.txt, each ffmpeg argv (the run's folders replaced by {dataset_folder}, {videos_folder} and
{ffmpeg_dir}), and a SHA-256 (pixel_sha256) of the decoded pixels of every blurry PNG and every sharp copy.
"""
import hashlib
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
OUT = os.path.join(REPO, "tests", "golden", "blur_tree.npz")
SCRIPT = os.path.join("data_scripts", "adobe240fps", "create_dataset_blur_N_frames_average.py")
LOG_ENV = "BLUR_TREE_FFMPEG_LOG"

VIDEOS = {"clip_a.mp4": (64, 2101), "clip_b.MOV": (41, 2102), "clip_c.mov": (97, 2103)}   # T a multiple of 8 and not
TEST = ["clip_a.mp4", "clip_b.MOV"]
TRAIN = ["clip_c.mov"]
RUNS = {"ws11": dict(window_size=11, img_width=640, img_height=352),
        "ws7": dict(window_size=7, img_width=53, img_height=37)}

BOOT = r"""
import runpy, sys, types
import numpy as np
try:
    from PIL import Image
    def imread(path):
        with Image.open(path) as im:
            return np.array(im)
    def imsave(path, arr):
        Image.fromarray(arr).save(path)
except ImportError:
    import cv2
    def imread(path):
        img = cv2.imread(path, cv2.IMREAD_UNCHANGED)
        return np.ascontiguousarray(img[:, :, ::-1]) if img.ndim == 3 else img
    def imsave(path, arr):
        assert cv2.imwrite(path, np.ascontiguousarray(arr[:, :, ::-1]) if arr.ndim == 3 else arr)
scipy, nd, misc = (types.ModuleType(n) for n in ("scipy", "scipy.ndimage", "scipy.misc"))
nd.imread, misc.imsave, scipy.ndimage, scipy.misc = imread, imsave, nd, misc
sys.modules.update({"scipy": scipy, "scipy.ndimage": nd, "scipy.misc": misc})
sys.argv = sys.argv[1:]
runpy.run_path(sys.argv[0], run_name="__main__")
"""


def stub_main(argv):
    """The stub ffmpeg: append argv to $BLUR_TREE_FFMPEG_LOG, then write VIDEOS[basename of -i]'s frames to the
    pattern given last, at the size of scale=W:H."""
    import cv2
    from oracle.trainset_oracle import synth_clip
    with open(os.environ[LOG_ENV], "a") as fh:
        fh.write(json.dumps(list(argv)) + "\n")
    T, seed = VIDEOS[os.path.basename(argv[argv.index("-i") + 1])]
    W, H = (int(v) for v in argv[argv.index("-vf") + 1][len("scale="):].split(":"))
    for k, img in enumerate(synth_clip(T, H, W, seed)):
        assert cv2.imwrite(argv[-1] % (k + 1), img)


def write_stub(bin_dir: str) -> str:
    """An executable `ffmpeg` in bin_dir that runs stub_main.  -> bin_dir."""
    os.makedirs(bin_dir, exist_ok=True)
    path = os.path.join(bin_dir, "ffmpeg")
    with open(path, "w") as fh:
        fh.write(f"#!{sys.executable}\nimport sys\nsys.path.insert(0, {REPO!r})\n"
                 "from oracle.make_golden_blur_tree import stub_main\nstub_main(sys.argv)\n")
    os.chmod(path, 0o755)
    return bin_dir


def write_lists(cwd: str) -> None:
    """./test_list.txt and adobe240fps/train_list.txt, as the script opens them (no trailing newline: it would read
    one more video named '')."""
    os.makedirs(os.path.join(cwd, "adobe240fps"), exist_ok=True)
    for path, videos in (("test_list.txt", TEST), (os.path.join("adobe240fps", "train_list.txt"), TRAIN)):
        with open(os.path.join(cwd, path), "w") as fh:
            fh.write("\n".join(videos))


def pixel_sha256(path: str) -> str:
    """SHA-256 of a PNG's decoded pixels (cv2.imread IMREAD_UNCHANGED) and their shape."""
    import cv2
    img = cv2.imread(path, cv2.IMREAD_UNCHANGED)
    assert img is not None, path
    return hashlib.sha256(repr(img.shape).encode() + np.ascontiguousarray(img).tobytes()).hexdigest()


def describe(root: str, argv_log: str, folders) -> dict:
    """What a run wrote under root: files, dirs, {list path: text}, argvs (folders: {placeholder: path}), and
    {path: pixel_sha256} of every PNG under test_blur, train_blur, test and train."""
    files, dirs, lists, shas = [], [], {}, {}
    for d, sub, names in os.walk(root):
        rel = os.path.relpath(d, root)
        dirs += [os.path.normpath(os.path.join(rel, s)) for s in sub]
        for n in names:
            p = os.path.normpath(os.path.join(rel, n))
            files.append(p)
            if p.endswith("_im_list.txt"):
                with open(os.path.join(d, n), "rb") as fh:
                    lists[p] = fh.read().decode()
            elif p.split(os.sep)[0] in ("test_blur", "train_blur", "test", "train"):
                shas[p] = pixel_sha256(os.path.join(d, n))
    argvs = []
    if os.path.exists(argv_log):
        with open(argv_log) as fh:
            for line in fh:
                a = json.loads(line)
                for key, path in folders.items():
                    a = [x.replace(path, "{" + key + "}") for x in a]
                argvs.append(a)
    return {"files": sorted(files), "dirs": sorted(dirs), "lists": lists, "argv": argvs, "sha": shas}


def main(ref_root):
    script = os.path.join(ref_root, SCRIPT)
    assert os.path.isfile(script), script
    rec = {}
    for run, opt in RUNS.items():
        with tempfile.TemporaryDirectory() as tmp:
            cwd, data, videos = (os.path.join(tmp, n) for n in ("cwd", "data", "videos"))
            os.makedirs(cwd)
            os.makedirs(videos)
            write_lists(cwd)
            bin_dir = write_stub(os.path.join(tmp, "bin"))
            log = os.path.join(tmp, "argv.jsonl")
            args = ["--ffmpeg_dir", bin_dir, "--dataset", "adobe240fps_blur", "--videos_folder", videos,
                    "--dataset_folder", data, "--img_width", str(opt["img_width"]), "--img_height",
                    str(opt["img_height"]), "--window_size", str(opt["window_size"]), "--enable_train", "1"]
            subprocess.run([sys.executable, "-c", BOOT, script] + args, cwd=cwd, check=True,
                           env=dict(os.environ, **{LOG_ENV: log}))
            d = describe(data, log, {"dataset_folder": data, "videos_folder": videos, "ffmpeg_dir": bin_dir})
        rec[run] = json.dumps({"options": opt, **d}, sort_keys=True)
        print(run, opt, len(d["files"]), "files,", len(d["sha"]), "hashed,", len(d["argv"]), "ffmpeg calls;",
              {k: v.count("\n") + 1 if v else 0 for k, v in d["lists"].items()})
    np.savez_compressed(OUT, **{k: np.array(v) for k, v in rec.items()})
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main(sys.argv[1])
