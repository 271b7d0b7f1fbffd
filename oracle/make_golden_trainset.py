"""Generate tests/golden/trainset.npz by EXECUTING THE REFERENCE'S OWN training-set loader (CPU; needs the reference
checkout with cv2 importable):

    python oracle/make_golden_trainset.py /path/to/BIN

``trainset_oracle.write_tree`` writes a synthetic tree into a temporary directory: the clips of
``trainset_oracle.CLIPS`` (72 and 80 sharp frames at 352x640, 72 at 360x656, one im_list that omits a blurry frame),
sharp frames from stored seeds, blurry frames from the pinned ``bin_oracle.blur_average``.  The unmodified
``data/BIN_dataset.py BINDataset`` is built on it after ``random.seed(seed)`` and sampled at indices ``ORDER``;
pass-through wrappers of ``random.randint`` / ``random.choice`` record every draw.  The fixture keeps no frames: the
listdir order, the keys in shuffled order, the draws, and a SHA-256 of each sample's LQs / GTenh / GTinp bytes, for
each lq_size of ``trainset_oracle.LQ_SIZES``, plus a SHA-256 of each clip's frames.
"""
import os
import random
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(os.path.dirname(HERE), "tests", "golden", "trainset.npz")
SEEDS = {"a": 7, "b": 8, "c": 9}
REPEATS = 3                       # ORDER = every index, three times: 18 samples (the GPU tests take up to 17)


def main(ref_root):
    sys.path.insert(0, os.path.dirname(HERE))
    sys.path.insert(0, ref_root)
    from data.BIN_dataset import BINDataset          # the reference itself
    from oracle import trainset_oracle as TO
    rec = {}
    with tempfile.TemporaryDirectory() as root:
        TO.write_tree(root)
        listdir = os.listdir(os.path.join(root, "train_blur"))
        rec["listdir"] = np.array(listdir)
        for folder, T, H, W, seed, omit in TO.CLIPS:
            sharp, blurry, _, _ = TO.clip_arrays(T, H, W, seed)
            rec[f"clip_{folder}_sha256"] = np.array([TO.sha256(sharp), TO.sha256(blurry)])
        drawn = []
        orig_randint, orig_choice = random.randint, random.choice

        def randint(a, b):
            v = orig_randint(a, b)
            drawn.append(v)
            return v

        def choice(seq):
            v = orig_choice(seq)
            drawn.append(v)
            return v

        for tag, (h, w) in TO.LQ_SIZES.items():
            opt = {"dataroot_GT": root, "dataroot_LQ": root, "data_type": "img", "LQ_size": [3, h, w], "name": "train"}
            random.seed(SEEDS[tag])
            ds = BINDataset(opt)
            keys = [p[3] for p in ds.all_paths]
            order = list(range(len(ds))) * REPEATS
            shas, draws = [], []
            random.randint, random.choice = randint, choice
            try:
                for i in order:
                    del drawn[:]
                    s = ds[i]
                    assert s["key"] == keys[i] and len(drawn) == 4
                    assert s["LQs"].shape == (6, 3, h, w) and s["GTinp"].shape == (5, 3, h, w)
                    draws.append(list(drawn))
                    shas.append([TO.sha256(s[k].numpy()) for k in ("LQs", "GTenh", "GTinp")])
            finally:
                random.randint, random.choice = orig_randint, orig_choice
            draws = np.array(draws)
            assert set(draws[:, 0]) == {0, 1} and set(draws[:, 3]) == {0, 1}, "seed must give both orders and flips"
            rec[f"{tag}_meta"] = np.array([h, w, SEEDS[tag]])
            rec[f"{tag}_keys"] = np.array(keys)
            rec[f"{tag}_order"] = np.array(order)
            rec[f"{tag}_draws"] = draws
            rec[f"{tag}_sha256"] = np.array(shas)
            print(tag, (h, w), len(keys), "windows", keys, "draws", draws.tolist())
    np.savez_compressed(OUT, **rec)
    print("wrote", OUT, os.path.getsize(OUT), "bytes; listdir", listdir)


if __name__ == "__main__":
    main(sys.argv[1])
