"""CPU checks of the demo driver (bin_b200.demo): its write plan against a restatement of demo.py:164-324's loop over a
listing with its existence checks, its arguments and yml keys, the union of the ranks' plans, and the refusal of an
output directory that already holds one of its files."""
import os

import pytest

from bin_b200 import BinB200Error, dist, demo as D

TIME_STEPS = [0.5, 0.25, 0.125, 0.1, 1.0, 3.0]


# ----------------------------------------------------------------------------- the write plan
def reference_writes(n, first, time_step):
    """demo.py:101, 152-153, 164-324 as written, over a folder of n blurry frames named first, first + 8, ... into an
    empty directory; the model's outputs are named (window index, output index).  -> [(name, what it holds)] in write
    order."""
    disk = {}
    written = []

    def imwrite(name, img):
        disk[name] = img
        written.append((name, img))

    N_frames = round(1 / time_step)
    time_offsets_all = [kk * 1.0 / N_frames for kk in range(1, int(N_frames), 1)]
    time_step = range(0, N_frames - 1)
    nframes = 6
    our_model = True
    frames = sorted(str(first + 8 * k).zfill(5) + ".png" for k in range(n))
    shift_file = 1
    offset_file = 0
    for index, frame in enumerate(frames):
        if index == 0:
            first_frame_num = int(frame[:-4])    # noqa: F841
        if index >= len(frames) - 1:
            break
        second_frame_num = int(int(frame[:-4]) + 8)
        first_gt_deblur = int(int(frame[:-4]) * shift_file + offset_file + 4)
        second_gt_deblur = int(second_frame_num * shift_file + offset_file + 4)
        first_gt_deblur_name = str(first_gt_deblur).zfill(5) + '.png'
        second_gt_deblur_name = str(second_gt_deblur).zfill(5) + '.png'
        interpolated_sharp_list = range(first_gt_deblur + 1, second_gt_deblur)
        if len(time_step) == 1:
            frame_indexs = [3]
            if our_model:
                if nframes == 6:
                    frame_indexs = [3]
        else:
            assert len(time_step) == len(time_offsets_all)
            frame_indexs = range(0, 7)
        for frame_time_step, frame_index in zip(time_step, frame_indexs):
            middle_frame_num = interpolated_sharp_list[frame_index]
            arguments_strOut = str(middle_frame_num).zfill(5) + '.png'
            if arguments_strOut not in disk:
                y_, x0_s, x1_s = (index, 13), (index, 8), (index, 12)
                imwrite(arguments_strOut, y_)
            if index < len(frames) - 2:
                if second_gt_deblur_name not in disk:
                    imwrite(second_gt_deblur_name, x1_s)
            if first_gt_deblur_name not in disk:
                imwrite(first_gt_deblur_name, x0_s)
    return written


def plan_writes(n, first, time_step, windows=None):
    out = []
    for i in (range(max(n - 1, 0)) if windows is None else windows):
        for k, names in D.demo_py_writes(i, n, time_step, first).items():
            out += [(name, (i, k)) for name in names]
    return out


@pytest.mark.parametrize("time_step", TIME_STEPS)
@pytest.mark.parametrize("n", range(1, 13))
def test_writes_match_demo_py(n, time_step):
    ref = reference_writes(n, 17, time_step)
    got = plan_writes(n, 17, time_step)
    assert len({name for name, _ in ref}) == len(ref)           # demo.py writes no name twice into a fresh directory
    assert len({name for name, _ in got}) == len(got)
    assert dict(got) == dict(ref)                                # the same files, each holding the same output
    assert [w for _, (w, _) in got] == [w for _, (w, _) in ref]  # window by window, in demo.py's order
    per_window = len(D.demo_py_steps(time_step))
    if per_window and n > 1:
        assert len(got) == (n - 1) * per_window + (n - 2) + 1


def test_steps_follow_round_of_the_inverse():
    assert D.demo_py_steps(0.5) == (3,)
    assert D.demo_py_steps(0.125) == tuple(range(7))
    assert D.demo_py_steps(0.25) == (0, 1, 2)
    assert D.demo_py_steps(0.1) == tuple(range(7))
    assert D.demo_py_steps(0.4) == (3,)                          # round(2.5) == 2
    assert D.demo_py_steps(1.0) == D.demo_py_steps(3.0) == ()
    for bad in (0.0, -0.5):
        with pytest.raises(BinB200Error, match="time_step"):
            D.demo_py_steps(bad)
    assert D.demo_py_writes(0, 5, 1.0) == {}
    with pytest.raises(BinB200Error, match="no window"):
        D.demo_py_writes(4, 5, 0.5)


def test_messages():
    got = D.demo_py_messages("/in", "/out", 0.5, "w.pth")
    assert got == ["We interp the 30 fps blurry video to 60 fps slow-motion video!", "In Data: /in ",
                   "Padding mode: 32", "Model path: Joint Model:w.pth", "Save images: /out", "interpolate middle frame"]
    got = D.demo_py_messages("/in", "/out", 0.125, "w.pth")
    assert got[0] == "We interp the 30 fps blurry video to 240 fps slow-motion video!"
    assert got[-1] == "interpolate all 7 frames"


# ----------------------------------------------------------------------------- sharding
@pytest.mark.parametrize("time_step", [0.5, 0.125])
@pytest.mark.parametrize("world", range(1, 5))
def test_rank_plans_cover_the_one_rank_plan(world, time_step):
    lengths = {"a": 2, "b": 7, "c": 1, "d": 3, "e": 12}
    whole = {(f, name): what for f, n in lengths.items() for name, what in plan_writes(n, 9, time_step)}
    union = {}
    for pieces in dist.shard_test_set(lengths, world):
        for f, rng in pieces:
            for name, what in plan_writes(lengths[f], 9, time_step, rng):
                assert (f, name) not in union                   # no file is written by two ranks
                union[(f, name)] = what
    assert union == whole


# ----------------------------------------------------------------------------- arguments and yml
YML = {"name": "bin_stage4", "distortion": "deblur",
       "network_G": {"which_model_G": "bin_stage4", "nframes": 6, "version": 2},
       "path": {"pretrain_model_G": "./model_weights/adobe_bin.pth", "strict_load": True}}


def test_demo_sh_arguments():
    args = D.parse_args(["--netName", "bin_stage4", "--input_path", "./demo_videos/demo_blur", "--output_path",
                         "./demo_videos/demo_results", "--time_step", "0.5", "--gpu_id", "2", "--opt",
                         "./options/train/train_adobe_stage4.yml"])
    assert (args.netName, args.input_path, args.output_path, args.time_step, args.gpu_id, args.opt) == (
        "bin_stage4", "./demo_videos/demo_blur", "./demo_videos/demo_results", 0.5, "2",
        "./options/train/train_adobe_stage4.yml")
    assert (args.weights, args.precision, args.flipx4, args.arch, args.decode_threads) == (None, "fp16", False, None, 8)
    args = D.parse_args(["--netName", "b", "--input_path", "i", "--output_path", "o", "--opt", "y", "--direct_interp",
                         "True", "--launcher", "pytorch", "--local_rank", "1", "--weights", "w.pth", "--precision",
                         "fp32", "--flipx4", "--arch", "64,6", "--decode_threads", "3"])
    assert (args.direct_interp, args.launcher, args.local_rank, args.weights, args.precision, args.flipx4, args.arch,
            args.decode_threads) == (True, "pytorch", 1, "w.pth", "fp32", True, (64, 6), 3)
    with pytest.raises(SystemExit):
        D.parse_args(["--netName", "b", "--input_path", "i", "--output_path", "o", "--opt", "y", "--arch", "64"])


def test_yml_keys(tmp_path):
    import copy
    import yaml
    p = tmp_path / "demo.yml"
    p.write_text(yaml.safe_dump(YML))
    opts = D.load_options(str(p))
    assert opts == D.DemoOptions("./model_weights/adobe_bin.pth", True)
    base = D.parse_args(["--netName", "b", "--input_path", "i", "--output_path", "o", "--opt", str(p)])
    assert D.weights_of(base, opts) == ("./model_weights/adobe_bin.pth", True)
    over = D.parse_args(["--netName", "b", "--input_path", "i", "--output_path", "o", "--opt", str(p), "--weights",
                         "mine.pth"])
    assert D.weights_of(over, opts) == ("mine.pth", True)
    loose = copy.deepcopy(YML)
    loose["path"]["strict_load"] = False
    assert D.weights_of(over, D.parse_options(loose)) == ("mine.pth", False)
    none = copy.deepcopy(YML)
    none["path"]["pretrain_model_G"] = None
    with pytest.raises(BinB200Error, match="path.pretrain_model_G"):
        D.weights_of(base, D.parse_options(none))
    assert D.weights_of(over, D.parse_options(none)) == ("mine.pth", True)
    for key, value, match in [("which_model_G", "bin_stage3", "network_G.which_model_G"),
                              ("which_model_G", None, "network_G.which_model_G"),
                              ("nframes", 5, "network_G.nframes"), ("nframes", None, "network_G.nframes")]:
        bad = copy.deepcopy(YML)
        if value is None:
            del bad["network_G"][key]
        else:
            bad["network_G"][key] = value
        with pytest.raises(BinB200Error, match=match):
            D.parse_options(bad)


def test_gpu_id():
    env = {}
    assert D.select_gpu("2", env) is None and env == {"CUDA_VISIBLE_DEVICES": "2"}
    env = {"WORLD_SIZE": "4"}
    msg = D.select_gpu("2", env)
    assert "ignored under torchrun" in msg and "CUDA_VISIBLE_DEVICES" not in env
    env = {}
    assert D.select_gpu(None, env) is None and env == {}


# ----------------------------------------------------------------------------- refusals
def make_listing(root, folders, first=17):
    for f, n in folders.items():
        os.makedirs(os.path.join(root, f))
        for k in range(n):
            open(os.path.join(root, f, str(first + 8 * k).zfill(5) + ".png"), "wb").close()


def tree(root):
    return sorted(os.path.relpath(os.path.join(d, f), root) for d, _, fs in os.walk(root) for f in fs)


def test_existing_output_raises_before_anything_runs(tmp_path):
    from bin_b200 import rdn
    net = rdn.bin_stage4_lstm().eval()
    inp, out = str(tmp_path / "in"), str(tmp_path / "out")
    make_listing(inp, {"a": 3, "b": 4})
    os.makedirs(os.path.join(out, "b"))
    open(os.path.join(out, "b", "00040.png"), "wb").close()     # window 2 of b, j = 2 under time_step 0.125
    before = tree(out)
    rdn.set_outputs(net, (13,))
    with pytest.raises(BinB200Error, match="00040.png exists"):
        D.run_demo(net, inp, out, time_step=0.125)
    assert tree(out) == before and not os.path.isdir(os.path.join(out, "a"))
    assert rdn._outputs_of(net)[0] == (13,)
    # the rank that runs folder b finds it too
    assert dist.shard_test_set({"a": 3, "b": 4}, 2)[1] == [("b", range(0, 3))]
    with pytest.raises(BinB200Error, match="00040.png exists"):
        D.run_demo(net, inp, out, time_step=0.125, rank=1, world=2)


def test_badly_named_folder_raises(tmp_path):
    from bin_b200 import rdn
    net = rdn.bin_stage4_lstm().eval()
    inp = str(tmp_path / "in")
    make_listing(inp, {"a": 3})
    open(os.path.join(inp, "a", "00030.png"), "wb").close()
    with pytest.raises(BinB200Error, match="run_demo: the blurry frames of a must be named"):
        D.run_demo(net, inp, str(tmp_path / "out"))
    with pytest.raises(BinB200Error, match="rank 2 is not in 0..1"):
        D.run_demo(net, inp, str(tmp_path / "out"), rank=2, world=2)


def test_no_step_runs_nothing(tmp_path, capsys):
    from bin_b200 import rdn
    net = rdn.bin_stage4_lstm().eval()                          # on the CPU: any window run would raise
    inp, out = str(tmp_path / "in"), str(tmp_path / "out")
    make_listing(inp, {"a": 3, "b": 4})
    stats = D.run_demo(net, inp, out, time_step=1.0)
    assert stats == D.DemoStats(0, 0, 0.0, 0.0)
    assert sorted(os.listdir(out)) == ["a", "b"] and tree(out) == []     # demo.py makes the folders all the same
    assert capsys.readouterr().out.splitlines()[-1] == "no window run: this time_step writes no image"
