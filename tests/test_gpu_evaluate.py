"""The test-set evaluator on the GPU: the batched metrics against the single-pair kernel and the skimage drop-ins,
stream_video over a range of windows against the net per window, and evaluate_testset end to end against a
restatement of test.py's loop (module call per window, cv2.imwrite, cv2 re-read, bin_b200.metrics drop-ins) on a
seeded PNG tree, at world 1, at world 3 emulated in one process, and at world 2 over NCCL when two GPUs are visible."""
import ctypes as C
import math
import os
import re

import numpy as np
import pytest
import torch

from oracle import arch_oracle as A
from oracle import bin_oracle as O

pytestmark = pytest.mark.gpu


# ----------------------------------------------------------------------------- batched metrics
def single(a, b):
    from bin_b200 import _lib
    L = _lib.lib()
    h, w = a.shape[:2]
    c = a.shape[2] if a.dim() == 3 else 1
    out = torch.empty(4, dtype=torch.float64, device="cuda")
    ws = torch.empty(max(int(L.bin_image_metrics_workspace_bytes(h, w)), 8), dtype=torch.uint8, device="cuda")
    _lib.check(L.bin_image_metrics_u8(a.data_ptr(), b.data_ptr(), h, w, c, out.data_ptr(), ws.data_ptr(), ws.numel(),
                                      torch.cuda.current_stream().cuda_stream))
    return out


def bits(t):
    return t.cpu().numpy().view(np.uint64)


@pytest.mark.parametrize("h,w", [(7, 7), (11, 13), (37, 53), (64, 96), (720, 1280)])
@pytest.mark.parametrize("c", [1, 3])
def test_batch_equals_single_calls(h, w, c):
    from bin_b200.metrics import image_metrics_batch
    g = np.random.default_rng(h * 7 + w + c)
    shape = (h, w, c) if c == 3 else (h, w)
    pool = [torch.from_numpy(g.integers(0, 256, size=shape, dtype=np.uint8)).cuda() for _ in range(6)]
    pool.append(((pool[0].int() + 1).clamp(max=255)).to(torch.uint8))        # close to pool[0]: high SSIM
    ns = range(1, 17) if h * w <= 64 * 96 else (1, 5, 16)
    for n in ns:
        pairs = [(pool[int(g.integers(0, 7))], pool[int(g.integers(0, 7))]) for _ in range(n)]   # shared operands
        got = image_metrics_batch(pairs)
        assert got.shape == (n, 4) and got.dtype == torch.float64
        want = torch.stack([single(a, b) for a, b in pairs])
        assert np.array_equal(bits(got), bits(want)), n


@pytest.mark.parametrize("h,w", [(7, 9), (48, 80), (720, 1280)])
def test_bgr_flag_scores_the_rgb_view(h, w):
    from bin_b200.metrics import compare_psnr, compare_ssim, image_metrics_batch
    g = np.random.default_rng(h + w)
    base = g.integers(0, 256, size=(h, w, 3), dtype=np.uint8)
    noisy = np.clip(base.astype(int) + g.integers(-20, 21, size=base.shape), 0, 255).astype(np.uint8)
    pairs = [(base, noisy), (noisy, base), (base, base[::-1].copy()), (noisy, noisy)]
    dev = [(torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()) for a, b in pairs]
    got = image_metrics_batch(dev, bgr=True).cpu().numpy()
    for (a, b), row, (da, db) in zip(pairs, got, dev):
        ra, rb = np.ascontiguousarray(a[:, :, ::-1]), np.ascontiguousarray(b[:, :, ::-1])      # read_image_np's view
        want = single(torch.from_numpy(ra).cuda(), torch.from_numpy(rb).cuda()).cpu().numpy()
        assert np.array_equal(row.view(np.uint64), want.view(np.uint64))
        assert row[3] == compare_ssim(ra, rb, multichannel=True)
        n = a.size
        psnr = np.float64(np.inf) if row[1] == 0 else 10 * np.log10((255 ** 2) / np.float64(int(row[1]) / n))
        assert psnr == compare_psnr(ra, rb)
    plain = image_metrics_batch(dev).cpu().numpy()
    assert np.array_equal(plain[:, :2], got[:, :2])            # the sums do not depend on the channel order


def test_slots_past_n_keep_their_sentinel():
    from bin_b200 import _lib
    L = _lib.lib()
    h, w, n = 40, 50, 3
    g = np.random.default_rng(3)
    imgs = [torch.from_numpy(g.integers(0, 256, size=(h, w, 3), dtype=np.uint8)).cuda() for _ in range(2)]
    out = torch.full((16, 4), -1234.5, dtype=torch.float64, device="cuda")
    ws = torch.empty(int(L.bin_image_metrics_batch_workspace_bytes(n, h, w)), dtype=torch.uint8, device="cuda")
    pa = (C.c_void_p * n)(*[imgs[0].data_ptr()] * n)
    pb = (C.c_void_p * n)(*[imgs[1].data_ptr()] * n)
    _lib.check(L.bin_image_metrics_batch_u8(pa, pb, n, h, w, 3, 0, out.data_ptr(), ws.data_ptr(), ws.numel(),
                                            torch.cuda.current_stream().cuda_stream))
    o = out.cpu()
    assert bool((o[n:] == -1234.5).all())
    assert np.array_equal(bits(o[:n]), bits(single(imgs[0], imgs[1]).cpu().expand(n, 4)))


# ----------------------------------------------------------------------------- stream_video over a range
@pytest.fixture(scope="module")
def nets():
    from bin_b200 import rdn
    net = rdn.bin_stage4_lstm()
    net.load_state_dict(O.synth_state_dict(0), strict=True)
    light = rdn.bin_stage4_lstm()
    light.model = rdn.RDN_residual_interp_5_input(lstm=True, GO=64, D=6)
    light.load_state_dict(A.synth_state_dict(0, 64, 6), strict=True)
    return {"shipped": net.cuda().eval(), "light": light.cuda().eval()}


@pytest.mark.parametrize("name", ["shipped", "light", "selection"])
@pytest.mark.parametrize("n", range(2, 10))
def test_range_stream_matches_the_net(nets, n, name):
    from bin_b200 import rdn
    from bin_b200.streaming import VideoPlan, stream_video, test_py_window
    net = nets["light" if name == "light" else "shipped"]
    if name == "selection":
        rdn.set_outputs(net, (13, 8, 12))
    try:
        video = [f.cuda() for f in O.synth_frames(n, 1, 32, 48, seed=40 + n, smooth=True)]
        with torch.no_grad():
            ref = [net(*[video[j] for j in test_py_window(i, n)]) for i in range(n - 1)]
        sel = rdn._outputs_of(net)
        live = rdn._window_live(range(14) if sel is None else sel[0])
        for a in range(n - 1):
            for b in range(a + 1, n):
                s = stream_video(net, iter(video[max(a - 2, 0):]), windows=range(a, b), n=n)
                got = list(s)
                assert [i for i, _ in got] == list(range(a, b))
                for i, o in got:
                    assert all((x is None and y is None) or torch.equal(x, y) for x, y in zip(o, ref[i])), (a, b, i)
                plan = VideoPlan(live, range(a, b), n)
                steps = []
                while not plan.complete:
                    steps += plan.arrive()
                assert s.backbone_calls == sum(st.backbone_calls for st in steps)
    finally:
        rdn.set_outputs(net, None)


# ----------------------------------------------------------------------------- end to end
FOLDERS = {"clipA": (2, 96, 160), "clipB": (5, 100, 130), "clipC": (9, 96, 160)}
FIRST = 17


def make_tree(root, seed):
    import cv2
    g = np.random.default_rng(seed)
    for folder, (n, h, w) in FOLDERS.items():
        for sub in ("in", "gt"):
            os.makedirs(os.path.join(root, sub, folder))
        last = FIRST + 8 * (n - 1) + 12
        base = g.integers(0, 256, size=(h // 4 + 2, w // 4 + 2, 3)).astype(np.float32)
        for num in range(FIRST, last + 1):
            shift = g.normal(0, 6, size=base.shape).astype(np.float32)
            img = cv2.resize(base + shift, (w, h), interpolation=cv2.INTER_LINEAR)
            gt = np.clip(np.round(img + g.normal(0, 3, size=img.shape)), 0, 255).astype(np.uint8)
            cv2.imwrite(os.path.join(root, "gt", folder, f"{num:05d}.png"), gt)
            if (num - FIRST) % 8 == 0 and (num - FIRST) // 8 < n:
                blur = cv2.GaussianBlur(gt, (7, 7), 2.0)
                cv2.imwrite(os.path.join(root, "in", folder, f"{num:05d}.png"), blur)
    return os.path.join(root, "in"), os.path.join(root, "gt")


def reference_run(net, input_path, gt_path, output_path, net_name, direct_interp):
    """test.py:158-506 restated: one module call per window, tensor2img, cv2.imwrite, cv2 re-read, the metric drop-ins.
    -> (log messages, summary messages) without the runtime line."""
    import cv2
    from bin_b200 import metrics as M
    from bin_b200.evaluate import AverageMeter
    compare_psnr = M.compare_psnr
    my_compare_ssim = lambda a, b: M.compare_ssim(a, b, multichannel=True)   # noqa: E731
    read_image_np = lambda p: cv2.imread(p)[:, :, [2, 1, 0]]                   # noqa: E731
    RESULT_PATH = os.path.join(output_path, "60fps_test_results")
    gen_dir = os.path.join(RESULT_PATH, net_name)
    os.makedirs(gen_dir, exist_ok=True)
    n_params = sum([np.prod(p.size()) for p in net.parameters() if p.requires_grad])
    pstring_model_size = 'Num. of model parameters is : {}'.format(str(n_params))
    log = ['In Data: {} '.format(input_path), 'Padding mode: 32', 'Model path: Joint Model:', 'Save images: ' + RESULT_PATH,
           'Flip test: False', 'Use ssin method skimage.measure.ssim', pstring_model_size]
    summ = []
    sets = [AverageMeter() for _ in range(7)]
    interp_error_set, psnr_interp_total_set, ssim_interp_total_set, psnr_deblur_total_set, ssim_deblur_total_set, \
        psnr_blurry_total_set, ssim_blurry_total_set = sets
    for dir in sorted(os.listdir(input_path)):
        interp_error, psnr_interp_total, ssim_interp_total, psnr_deblur_total, ssim_deblur_total, psnr_blurry_total, \
            ssim_blurry_total = [AverageMeter() for _ in range(7)]
        os.makedirs(os.path.join(gen_dir, dir), exist_ok=True)
        log.append("The results for dir:{}".format(dir))
        summ.append("The results for dir:{}".format(dir))
        frames_path, sharp_path = os.path.join(input_path, dir), os.path.join(gt_path, dir)
        frames = sorted(os.listdir(frames_path))
        for index, frame in enumerate(frames):
            if index == 0:
                first_frame_num = int(frame[:-4])
            if index >= len(frames) - 1:
                break
            L = len(frames) - 1
            first_5 = [8 * k for k in [max(index - 2, 0), max(index - 1, 0), min(index, L), min(index + 1, L), min(index + 2, L)]]
            second_5 = [8 * k for k in [max(index - 1, 0), max(index, 0), min(index + 1, L), min(index + 2, L), min(index + 3, L)]]
            src = sharp_path if direct_interp else frames_path
            strFirst = [os.path.join(src, str(first_frame_num + i).zfill(5) + '.png') for i in first_5]
            strSecond = [os.path.join(src, str(first_frame_num + i).zfill(5) + '.png') for i in second_5]
            first_gt_deblur = int(frame[:-4]) + 4
            second_gt_deblur = int(frame[:-4]) + 8 + 4
            first_gt_deblur_name = str(first_gt_deblur).zfill(5) + '.png'
            second_gt_deblur_name = str(second_gt_deblur).zfill(5) + '.png'
            first_blurry_path = strSecond[2]
            middle_frame_name = str(range(first_gt_deblur + 1, second_gt_deblur)[3]).zfill(5) + '.png'
            out_mid = os.path.join(gen_dir, dir, middle_frame_name)
            gt_middle_path = os.path.join(gt_path, dir, middle_frame_name)
            out_first = os.path.join(gen_dir, dir, first_gt_deblur_name)
            out_second = os.path.join(gen_dir, dir, second_gt_deblur_name)
            imgs = [cv2.imread(p) for p in strFirst[:5] + [strSecond[4]]]
            h, w = imgs[0].shape[:2]
            from bin_b200.streaming import test_py_padding
            pl, pr, pt, pb = test_py_padding(h, w)
            pader = torch.nn.ReplicationPad2d([pl, pr, pt, pb])
            data = [pader(O.read_image_u8(im).unsqueeze(0)).cuda() for im in imgs]
            with torch.no_grad():
                Ft_p = net(*data)
            crop = lambda t: O.tensor2img_bgr_u8(t.squeeze(0).cpu())[pt:pt + h, pl:pl + w, :]   # noqa: E731
            y_, x0_s, x1_s = crop(Ft_p[13]), crop(Ft_p[8]), crop(Ft_p[12])
            cv2.imwrite(out_mid, y_)
            if index < len(frames) - 2 and not os.path.exists(out_second):
                cv2.imwrite(out_second, x1_s)
                gt = read_image_np(os.path.join(gt_path, dir, second_gt_deblur_name))
                res = read_image_np(out_second)
                psnr_tmp, ssim_tmp = compare_psnr(res, gt), my_compare_ssim(res, gt)
                psnr_deblur_total.update(psnr_tmp, 1)
                ssim_deblur_total.update(ssim_tmp, 1)
                log.append("Interp PSNR : " + str(round(psnr_tmp, 4)) + " Interp SSIM : " + str(round(ssim_tmp, 4)))
            if not os.path.exists(out_first):
                cv2.imwrite(out_first, x0_s)
                gt = read_image_np(os.path.join(gt_path, dir, first_gt_deblur_name))
                res = read_image_np(out_first)
                psnr_tmp, ssim_tmp = compare_psnr(res, gt), my_compare_ssim(res, gt)
                psnr_deblur_total.update(psnr_tmp, 1)
                ssim_deblur_total.update(ssim_tmp, 1)
                log.append("Interp PSNR : " + str(round(psnr_tmp, 4)) + " Interp SSIM : " + str(round(ssim_tmp, 4)))
            rec_rgb, gt_rgb = read_image_np(out_mid), read_image_np(gt_middle_path)
            diff_rgb = 128.0 + rec_rgb - gt_rgb
            avg_interp_error_abs = np.mean(np.abs(diff_rgb - 128.0))
            interp_error.update(avg_interp_error_abs, 1)
            mse = np.mean((diff_rgb - 128.0) ** 2)
            assert mse != 0
            psnr = 20 * math.log10(255.0 / math.sqrt(mse))
            ssim_tmp = my_compare_ssim(rec_rgb, gt_rgb)
            psnr_interp_total.update(psnr, 1)
            ssim_interp_total.update(ssim_tmp, 1)
            log.append("deblur error / PSNR : " + str(round(avg_interp_error_abs, 4)) + " / " + str(round(psnr, 4)))
            blur = read_image_np(first_blurry_path)
            psnr_tmp, ssim_tmp = compare_psnr(blur, gt_rgb), my_compare_ssim(blur, gt_rgb)
            psnr_blurry_total.update(psnr_tmp, 1)
            ssim_blurry_total.update(ssim_tmp, 1)
            log.append("blurry PSNR : " + str(round(psnr_tmp, 4)) + " blurry SSIM : " + str(round(ssim_tmp, 4)) + '\n'
                       + first_blurry_path)
        summ.append("The results for dir:" + dir)
        summ.append("The average interpolation error " + str(round(interp_error.avg, 4)))
        summ.append("Avg. folder" + " blurry psnr " + str(psnr_blurry_total.avg) + " deblur psnr " + str(psnr_interp_total.avg)
                    + " interp psnr " + str(psnr_deblur_total.avg) + " blurry ssim " + str(ssim_blurry_total.avg)
                    + " deblur ssim " + str(ssim_interp_total.avg) + " interp ssim " + str(ssim_deblur_total.avg))
        for s, v in zip(sets, (interp_error, psnr_interp_total, ssim_interp_total, psnr_deblur_total, ssim_deblur_total,
                               psnr_blurry_total, ssim_blurry_total)):
            s.update(v.avg, 1)
    summ.append("The results for Adobe dataset")
    summ.append("The average interpolation error " + str(round(interp_error_set.avg, 4)))
    summ.append("Avg. testset " + " interp psnr " + str(psnr_deblur_total_set.avg) + " blurry psnr"
                + str(psnr_blurry_total_set.avg) + " deblur psnr" + str(psnr_interp_total_set.avg) + " interp ssim "
                + str(ssim_deblur_total_set.avg) + " blurry ssim" + str(ssim_blurry_total_set.avg) + " deblur ssim"
                + str(ssim_interp_total_set.avg))
    summ.append(pstring_model_size)
    return log, summ


_PREFIX = re.compile(r"^\d\d-\d\d-\d\d \d\d:\d\d:\d\d\.\d\d\d - INFO: ", re.M)


def read_logs(gen_dir):
    out = []
    for kind in ("test_", "test_summary_"):
        names = [f for f in os.listdir(gen_dir) if re.fullmatch(kind + r"\d{6}-\d{6}\.log", f)]
        assert len(names) == 1, names
        text = open(os.path.join(gen_dir, names[0])).read()
        msgs = [m[:-1] if m.endswith("\n") else m for m in _PREFIX.split(text)[1:]]
        out.append([m for m in msgs if not m.startswith("runtime per image [s] : ")])
    return tuple(out)


def tree_files(root):
    return sorted(os.path.relpath(os.path.join(d, f), root) for d, _, fs in os.walk(root) for f in fs if f.endswith(".png"))


class _Done(Exception):
    pass


def run_world(monkeypatch, net, inp, gt, out, world, direct_interp):
    from bin_b200 import evaluate as E
    got = {}
    for rank in reversed(range(world)):
        def fake_gather(local, w, rank=rank):
            got[rank] = local
            if rank != 0:
                raise _Done
            return [got[r] for r in range(w)]
        monkeypatch.setattr(E, "_gather", fake_gather)
        if rank == 0:
            E.evaluate_testset(net, inp, gt, out, "bin", direct_interp=direct_interp, rank=0, world=world, decode_threads=3)
        else:
            with pytest.raises(_Done):
                E.evaluate_testset(net, inp, gt, out, "bin", direct_interp=direct_interp, rank=rank, world=world)


@pytest.mark.parametrize("direct_interp", [False, True])
def test_evaluator_matches_test_py(nets, tmp_path, monkeypatch, direct_interp):
    import cv2
    from bin_b200 import BinB200Error, rdn
    net = nets["shipped"]
    inp, gt = make_tree(str(tmp_path / "data"), seed=11)
    ref_out = str(tmp_path / "ref")
    rdn.set_outputs(net, (13, 8, 12))
    try:
        ref = reference_run(net, inp, gt, ref_out, "bin", direct_interp)
    finally:
        rdn.set_outputs(net, None)
    ref_dir = os.path.join(ref_out, "60fps_test_results", "bin")
    ref_files = tree_files(ref_dir)
    assert len(ref_files) == sum(2 * n - 2 for n, _, _ in FOLDERS.values())   # Ft_p[13] and [12] per window, one [8]
    for world in (1, 3):
        out = str(tmp_path / f"w{world}")
        run_world(monkeypatch, net, inp, gt, out, world, direct_interp)
        assert rdn._outputs_of(net) is None                 # the caller's selection is restored
        gen = os.path.join(out, "60fps_test_results", "bin")
        assert tree_files(gen) == ref_files
        for f in ref_files:
            a, b = cv2.imread(os.path.join(ref_dir, f)), cv2.imread(os.path.join(gen, f))
            assert a is not None and np.array_equal(a, b), f
        log, summ = read_logs(gen)
        assert log == [m.replace(ref_out, out) for m in ref[0]]        # "Save images:" names the output directory
        assert summ == ref[1]
    # a second run into the same directory would resume: refused
    monkeypatch.undo()
    from bin_b200 import evaluate as E
    with pytest.raises(BinB200Error, match="exists"):
        E.evaluate_testset(net, inp, gt, str(tmp_path / "w1"), "bin", direct_interp=direct_interp)


def _nccl_worker(rank, world, inp, gt, out, port):
    import torch.distributed as tdist
    from bin_b200 import evaluate as E, rdn
    torch.cuda.set_device(rank)
    tdist.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    try:
        net = rdn.bin_stage4_lstm()
        net.load_state_dict(O.synth_state_dict(0), strict=True)
        net = net.cuda().eval()
        E.evaluate_testset(net, inp, gt, out, "bin")
    finally:
        tdist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_processes_over_nccl(nets, tmp_path):
    import socket
    import torch.multiprocessing as mp
    from bin_b200 import evaluate as E
    inp, gt = make_tree(str(tmp_path / "data"), seed=12)
    E.evaluate_testset(nets["shipped"], inp, gt, str(tmp_path / "w1"), "bin")
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    mp.spawn(_nccl_worker, args=(2, inp, gt, str(tmp_path / "w2"), port), nprocs=2, join=True)
    g1 = os.path.join(str(tmp_path / "w1"), "60fps_test_results", "bin")
    g2 = os.path.join(str(tmp_path / "w2"), "60fps_test_results", "bin")
    assert tree_files(g1) == tree_files(g2)
    assert read_logs(g1) == read_logs(g2)
