"""The demo driver on the GPU: run_demo against a restatement of demo.py's loop (one module call per window and per j
through the caller harness: read, pad, test_set_input / test_forward, crop, tensor2img, cv2.imwrite) on seeded folders
of 2, 3 and 7 frames at 128x256 and 90x130, at world 1 and 3 emulated in one process, for time_step 0.5 and 0.125, in
the default mode, the fp32 mode, with flip-x4 and on a light window; and python -m bin_b200.demo once end to end."""
import os

import numpy as np
import pytest
import torch

from caller_harness import CallerModel, pad_like_test_py, tensor2img
from oracle import arch_oracle as A
from oracle import bin_oracle as O

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FOLDERS = {"clipA": (2, 128, 256), "clipB": (3, 90, 130), "clipC": (7, 128, 256)}     # frames, height, width
FIRST = 17


@pytest.fixture(scope="module")
def nets():
    from bin_b200 import rdn
    net = rdn.bin_stage4_lstm()
    net.load_state_dict(O.synth_state_dict(0), strict=True)
    light = rdn.bin_stage4_lstm()
    light.model = rdn.RDN_residual_interp_5_input(lstm=True, GO=64, D=6)
    light.load_state_dict(A.synth_state_dict(0, 64, 6), strict=True)
    return {"shipped": net.cuda().eval(), "light": light.cuda().eval()}


@pytest.fixture(scope="module")
def blurry(tmp_path_factory):
    import cv2
    root = str(tmp_path_factory.mktemp("demo") / "in")
    g = np.random.default_rng(21)
    for folder, (n, h, w) in FOLDERS.items():
        os.makedirs(os.path.join(root, folder))
        base = g.integers(0, 256, size=(h // 4 + 2, w // 4 + 2, 3)).astype(np.float32)
        for k in range(n):
            img = cv2.resize(base + g.normal(0, 6, size=base.shape).astype(np.float32), (w, h),
                             interpolation=cv2.INTER_LINEAR)
            img = cv2.GaussianBlur(np.clip(np.round(img), 0, 255).astype(np.uint8), (7, 7), 2.0)
            cv2.imwrite(os.path.join(root, folder, f"{FIRST + 8 * k:05d}.png"), img)
    return root


def read_image(img_path):
    """demo.py:32-44."""
    import cv2
    img_GT = cv2.imread(img_path)
    img = img_GT.astype(np.float32) / 255.
    img = img[:, :, [2, 1, 0]]
    return torch.from_numpy(np.ascontiguousarray(np.transpose(img, (2, 0, 1)))).float()


def reference_run(net, input_path, output_path, time_step):
    """demo.py:101-324 restated: one module call per window and per j, through the caller harness's steps."""
    import cv2
    model = CallerModel(net, "cuda:0", device_ids=[0])
    N_frames = round(1 / time_step)
    time_offsets_all = [kk * 1.0 / N_frames for kk in range(1, int(N_frames), 1)]
    time_step = range(0, N_frames - 1)
    gen_dir = output_path
    os.makedirs(gen_dir, exist_ok=True)
    for dir in sorted(os.listdir(input_path)):
        os.makedirs(os.path.join(gen_dir, dir), exist_ok=True)
        frames_path = os.path.join(input_path, dir)
        frames = sorted(os.listdir(frames_path))
        for index, frame in enumerate(frames):
            if index == 0:
                first_frame_num = int(frame[:-4])
            if index >= len(frames) - 1:
                break
            L = len(frames) - 1
            first_5 = [8 * k for k in [max(index - 2, 0), max(index - 1, 0), min(index, L), min(index + 1, L), min(index + 2, L)]]
            second_5 = [8 * k for k in [max(index - 1, 0), max(index, 0), min(index + 1, L), min(index + 2, L), min(index + 3, L)]]
            strFirst = [os.path.join(frames_path, str(first_frame_num + i).zfill(5) + '.png') for i in first_5]
            strSecond = [os.path.join(frames_path, str(first_frame_num + i).zfill(5) + '.png') for i in second_5]
            first_gt_deblur = int(frame[:-4]) + 4
            second_gt_deblur = int(frame[:-4]) + 8 + 4
            first_path = os.path.join(gen_dir, dir, str(first_gt_deblur).zfill(5) + '.png')
            second_path = os.path.join(gen_dir, dir, str(second_gt_deblur).zfill(5) + '.png')
            interpolated_sharp_list = range(first_gt_deblur + 1, second_gt_deblur)
            if len(time_step) == 1:
                frame_indexs = [3]
            else:
                assert len(time_step) == len(time_offsets_all)
                frame_indexs = range(0, 7)
            for _, frame_index in zip(time_step, frame_indexs):
                out_path = os.path.join(gen_dir, dir, str(interpolated_sharp_list[frame_index]).zfill(5) + '.png')
                testData = [read_image(p).to("cuda:0") for p in strFirst + [strSecond[4]]]
                H, W = testData[0].size(1), testData[0].size(2)
                testData, (pl, pr, pt, pb) = pad_like_test_py(testData)
                testData.append(torch.unsqueeze(torch.tensor(frame_index), 0))
                if not os.path.exists(out_path):
                    with torch.no_grad():
                        model.test_set_input(testData)
                        model.test_forward()
                    crop = lambda t: tensor2img(t.squeeze(0))[pt:pt + H, pl:pl + W, :]    # noqa: E731
                    y_, x0_s, x1_s = crop(model.Ft_p[13]), crop(model.Ft_p[8]), crop(model.Ft_p[12])
                    cv2.imwrite(out_path, y_)
                if index < len(frames) - 2 and not os.path.exists(second_path):
                    cv2.imwrite(second_path, x1_s)
                if not os.path.exists(first_path):
                    cv2.imwrite(first_path, x0_s)


def tree_files(root):
    return sorted(os.path.relpath(os.path.join(d, f), root) for d, _, fs in os.walk(root) for f in fs)


def assert_same_images(ref_dir, got_dir):
    import cv2
    files = tree_files(ref_dir)
    assert tree_files(got_dir) == files
    for f in files:
        a, b = cv2.imread(os.path.join(ref_dir, f)), cv2.imread(os.path.join(got_dir, f))
        assert a is not None and np.array_equal(a, b), f


def assert_copies_identical(out, time_step):
    from bin_b200.demo import demo_py_writes
    for folder, (n, _, _) in FOLDERS.items():
        for i in range(n - 1):
            names = demo_py_writes(i, n, time_step, FIRST)[13]
            data = {open(os.path.join(out, folder, f), "rb").read() for f in names}
            assert len(data) == 1, (folder, i)


def run_world(monkeypatch, net, inp, out, world, time_step):
    from bin_b200 import demo as D
    monkeypatch.setattr(D, "_gather", lambda local, w: [local])
    windows = 0
    for rank in range(world):
        windows += D.run_demo(net, inp, out, time_step=time_step, rank=rank, world=world, decode_threads=3).windows
    return windows


@pytest.mark.parametrize("time_step", [0.5, 0.125])
@pytest.mark.parametrize("mode", ["fp16", "fp32", "flipx4", "light"])
def test_demo_matches_demo_py(nets, blurry, tmp_path, monkeypatch, mode, time_step):
    from bin_b200 import rdn
    net = nets["light" if mode == "light" else "shipped"]
    rdn.set_precision(net, "fp32" if mode == "fp32" else "fp16")
    rdn.set_self_ensemble(net, "flipx4" if mode == "flipx4" else None)
    try:
        ref = str(tmp_path / "ref")
        reference_run(net, blurry, ref, time_step)
        per_window = 1 if time_step == 0.5 else 7
        assert len(tree_files(ref)) == sum((n - 1) * per_window + n - 1 for n, _, _ in FOLDERS.values())
        for world in (1, 3):
            out = str(tmp_path / f"w{world}")
            sel = None if world == 1 else (12,)
            rdn.set_outputs(net, sel)
            assert run_world(monkeypatch, net, blurry, out, world, time_step) == sum(n - 1 for n, _, _ in FOLDERS.values())
            assert (rdn._outputs_of(net) or (None,))[0] == sel       # the caller's selection is restored
            rdn.set_outputs(net, None)
            assert_same_images(ref, out)
            assert_copies_identical(out, time_step)
    finally:
        rdn.set_outputs(net, None)
        rdn.set_precision(net, "fp16")
        rdn.set_self_ensemble(net, None)


def test_command_line(blurry, tmp_path, monkeypatch):
    import subprocess
    import sys
    import yaml
    from bin_b200 import BinB200Error, demo as D, rdn
    weights = str(tmp_path / "w.pth")
    torch.save({"module." + k: v for k, v in O.synth_state_dict(0).items()}, weights)
    yml = str(tmp_path / "demo.yml")
    with open(yml, "w") as fh:
        yaml.safe_dump({"name": "bin_stage4", "network_G": {"which_model_G": "bin_stage4", "nframes": 6, "version": 2},
                        "path": {"pretrain_model_G": weights, "strict_load": True}}, fh)
    out = str(tmp_path / "cli")
    r = subprocess.run([sys.executable, "-m", "bin_b200.demo", "--netName", "bin_stage4", "--input_path", blurry,
                        "--output_path", out, "--time_step", "0.125", "--gpu_id", "0", "--opt", yml], cwd=ROOT,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = r.stdout.splitlines()
    assert lines[:6] == D.demo_py_messages(blurry, out, 0.125, weights)
    assert "windows/s" in lines[-1] and lines[-1].startswith("9 windows, 72 images on 1 GPU(s)"), lines[-1]
    net = rdn.bin_stage4_lstm()
    net.load_state_dict(O.synth_state_dict(0), strict=True)
    net = net.cuda().eval()
    lib = str(tmp_path / "lib")
    D.run_demo(net, blurry, lib, time_step=0.125, verbose=False)
    assert_same_images(lib, out)
    with pytest.raises(BinB200Error, match="exists"):
        D.run_demo(net, blurry, out, time_step=0.125, verbose=False)
