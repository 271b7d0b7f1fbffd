"""CPU checks of the test-set evaluator (bin_b200.evaluate): shard_test_set's cover and balance, VideoPlan over a range
of windows against the whole-video plan, the evaluator's file names against a restatement of test.py:249-320, and its
log messages from synthetic metric sums against a restatement of test.py's accumulation (test.py:404-506)."""
import math
import os

import numpy as np
import pytest

from bin_b200 import BinB200Error, dist, evaluate as E, streaming as S
from bin_b200.rdn import _window_live

FULL = _window_live(range(14))
SEL = _window_live((8, 12, 13))


# ----------------------------------------------------------------------------- shard_test_set
@pytest.mark.parametrize("lengths", [[1], [2], [3], [50], [2, 5, 9], [1, 50, 3, 2], [50, 50, 1], [3, 1, 1, 2]])
@pytest.mark.parametrize("world", range(1, 17))
def test_shard_test_set_covers_in_order(lengths, world):
    names = {f"f{k:02d}": n for k, n in enumerate(lengths)}
    shards = dist.shard_test_set(dict(reversed(list(names.items()))), world)     # any key order: folders are sorted
    assert len(shards) == world
    want = [(f, i) for f in sorted(names) for i in range(max(names[f] - 1, 0))]
    got = [(f, i) for pieces in shards for f, rng in pieces for i in rng]
    assert got == want
    sizes = [sum(len(r) for _, r in pieces) for pieces in shards]
    assert max(sizes) - min(sizes) <= 1
    for pieces in shards:
        assert all(len(r) > 0 and r.step == 1 for _, r in pieces)
        assert len({f for f, _ in pieces}) == len(pieces)


# ----------------------------------------------------------------------------- VideoPlan over a range
def run_range(live, n, rng, give_n=True):
    plan = S.VideoPlan(live, rng, n if give_n else None)
    steps, arrived = [], []
    while not plan.complete and plan.next_pos < n:
        arrived.append(plan.next_pos)
        steps += plan.arrive()
    if not plan.complete:
        steps += plan.end()
    return steps, arrived


def full_plan(live, n):
    plan = S.VideoPlan(live)
    steps = []
    for _ in range(n):
        steps += plan.arrive()
    return steps + plan.end()


@pytest.mark.parametrize("n", range(2, 13))
@pytest.mark.parametrize("live", [FULL, SEL], ids=["all14", "sel"])
def test_range_plan_matches_full_plan(n, live):
    full = full_plan(live, n)
    later = sum(1 for nd in live if nd[0] in (2, 3, 4))
    for a in range(n - 1):
        for b in range(a + 1, n):
            steps, arrived = run_range(live, n, range(a, b))
            assert [s.i for s in steps] == list(range(a, b))
            assert [s.frames for s in steps] == [f.frames for f in full[a:b]]
            assert arrived == list(range(max(a - 2, 0), min(b + 2, n - 1) + 1))
            # every live pair is evaluated once, the first time the range reads it
            live1 = [p for p in range(5) if (1, p) in live]
            pairs = {(s.frames[p], s.frames[p + 1]) for s in steps for p in live1}
            assert sum(s.backbone_calls for s in steps) == len(pairs) + later * (b - a)
            assert [p for s in steps for p in s.fresh] == list(dict.fromkeys(
                (s.frames[p], s.frames[p + 1]) for s in steps for p in live1))
            if live is FULL and a >= 2 and b - 1 <= n - 4:
                assert sum(s.backbone_calls for s in steps) == 12 * (b - a) + (b - a + 4)
            # every frame and pair is dropped by the range's last window, each once
            assert sorted(p for s in steps for p in s.evict_frames) == arrived
            assert sorted(p for s in steps for p in s.evict_pairs) == sorted(pairs)
            # n is needed only when a window reads a clamped end frame
            if b - 1 <= n - 4:
                steps2, _ = run_range(live, n, range(a, b), give_n=False)
                assert steps2 == steps
            else:
                with pytest.raises(BinB200Error, match="length n is needed"):
                    run_range(live, n, range(a, b), give_n=False)
    assert run_range(live, n, range(0, n - 1))[0] == full


def test_range_plan_rejects_bad_ranges():
    for bad in (range(0, 0), range(3, 1), range(-1, 2), range(0, 4, 2), [0, 1]):
        with pytest.raises(BinB200Error, match="non-empty range"):
            S.VideoPlan(FULL, bad)
    with pytest.raises(BinB200Error, match="not among them"):
        S.VideoPlan(FULL, range(0, 5), 5)


# ----------------------------------------------------------------------------- names
def reference_paths(input_path, gt_path, gen_dir, folder, n, first, direct_interp):
    """test.py:242-334 as written, for a folder of n blurry frames named first, first + 8, ...; `our_model` is True."""
    our_model = True
    frames_path = os.path.join(input_path, folder)
    sharp_path = os.path.join(gt_path, folder)
    frames = [str(first + 8 * k).zfill(5) + ".png" for k in range(n)]
    shift_file, offset_file = 1, 0
    out = []
    for index, frame in enumerate(frames):
        if index == 0:
            first_frame_num = int(frame[:-4])
        if index >= len(frames) - 1:
            break
        first_5_blurry_list = [max(index - 2, 0), max(index - 1, 0), min(index, len(frames) - 1),
                               min(index + 1, len(frames) - 1), min(index + 2, len(frames) - 1)]
        second_5_blurry_list = [max(index - 1, 0), max(index - 0, 0), min(index + 1, len(frames) - 1),
                                min(index + 2, len(frames) - 1), min(index + 3, len(frames) - 1)]
        first_5_blurry_list = [i * 8 for i in first_5_blurry_list]
        second_5_blurry_list = [i * 8 for i in second_5_blurry_list]
        arguments_strFirst = []
        for i in first_5_blurry_list:
            tmp_num_name = str(int(first_frame_num + i)).zfill(5) + '.png'
            if our_model and direct_interp == True:  # noqa: E712
                arguments_strFirst.append(os.path.join(sharp_path, tmp_num_name))
            else:
                arguments_strFirst.append(os.path.join(frames_path, tmp_num_name))
        arguments_strSecond = []
        for i in second_5_blurry_list:
            tmp_num_name = str(int(first_frame_num + i)).zfill(5) + '.png'
            if our_model and direct_interp == True:  # noqa: E712
                arguments_strSecond.append(os.path.join(sharp_path, tmp_num_name))
            else:
                arguments_strSecond.append(os.path.join(frames_path, tmp_num_name))
        second_frame_num = int(int(frame[:-4]) + 8)
        first_gt_deblur = int(int(frame[:-4]) * shift_file + offset_file + 4)
        second_gt_deblur = int(second_frame_num * shift_file + offset_file + 4)
        first_gt_deblur_name = str(first_gt_deblur).zfill(5) + '.png'
        second_gt_deblur_name = str(second_gt_deblur).zfill(5) + '.png'
        interpolated_sharp_list = range(first_gt_deblur + 1, second_gt_deblur)
        first_blurry_path = arguments_strSecond[2]
        middle_frame_name = str(interpolated_sharp_list[3]).zfill(5) + '.png'
        arguments_strOut = os.path.join(gen_dir, folder, middle_frame_name)
        gt_middle_path = os.path.join(gt_path, folder, middle_frame_name)
        first_gt_deblur_path = os.path.join(gt_path, folder, first_gt_deblur_name)
        second_gt_deblur_path = os.path.join(gt_path, folder, second_gt_deblur_name)
        list_tmp = [arguments_strFirst[0], arguments_strFirst[1], arguments_strFirst[2], arguments_strFirst[3],
                    arguments_strFirst[4], arguments_strSecond[4]]
        out.append((tuple(list_tmp), {13: gt_middle_path, 8: first_gt_deblur_path, 12: second_gt_deblur_path},
                    {13: arguments_strOut, 8: os.path.join(gen_dir, folder, first_gt_deblur_name),
                     12: os.path.join(gen_dir, folder, second_gt_deblur_name)}, first_blurry_path))
    return out


@pytest.mark.parametrize("n", range(1, 13))
@pytest.mark.parametrize("direct_interp", [False, True])
def test_window_paths_match_test_py(n, direct_interp):
    args = ("/data/in", "/data/gt", "/out/60fps_test_results/bin", "720p_240fps_1")
    ref = reference_paths(*args, n, 17, direct_interp)
    got = [tuple(E.window_paths(*args, 17, i, n, direct_interp)) for i in range(max(n - 1, 0))]
    assert got == ref


# ----------------------------------------------------------------------------- logs
class RefMeter:
    """utils/AverageMeter.py as written."""

    def __init__(self):
        self.reset()

    def reset(self):
        self.val = 0
        self.avg = 0
        self.sum = 0
        self.count = 0

    def update(self, val, n=1):
        self.val = val
        self.sum += val * n
        self.count += n
        self.avg = self.sum / self.count


def reference_logs(header, folders, sums, model_size, runtime, blurry_path):
    """test.py:190-506 as written, with each image pair's metric replaced by its synthetic sums: compare_psnr and
    my_compare_ssim as skimage computes them from (sum |a-b|, sum (a-b)^2, -, box SSIM), test.py's own PSNR from the
    mean of the exact squares.  -> (log messages after the header, summary messages, returned early)."""
    log, summ = [], []
    logger = type("L", (), {"info": staticmethod(log.append)})
    logger_summary = type("L", (), {"info": staticmethod(summ.append)})
    interp_error, psnr_interp_total, ssim_interp_total = RefMeter(), RefMeter(), RefMeter()
    psnr_deblur_total, ssim_deblur_total, psnr_blurry_total, ssim_blurry_total = RefMeter(), RefMeter(), RefMeter(), RefMeter()
    interp_error_set, psnr_interp_total_set, ssim_interp_total_set = RefMeter(), RefMeter(), RefMeter()
    psnr_deblur_total_set, ssim_deblur_total_set = RefMeter(), RefMeter()
    psnr_blurry_total_set, ssim_blurry_total_set = RefMeter(), RefMeter()

    def compare_psnr(pair):
        err = np.float64(pair["sq"] / pair["n"])
        return np.float64(np.inf) if err == 0 else 10 * np.log10((255 ** 2) / err)

    def my_compare_ssim(pair):
        return np.float64(pair["box"])

    for dir, n in folders:
        interp_error.reset(); psnr_interp_total.reset(); ssim_interp_total.reset()          # noqa: E702
        psnr_deblur_total.reset(); ssim_deblur_total.reset()                                # noqa: E702
        psnr_blurry_total.reset(); ssim_blurry_total.reset()                                # noqa: E702
        logger.info("The results for dir:{}".format(dir))
        logger_summary.info("The results for dir:{}".format(dir))
        for index in range(n):
            if index >= n - 1:
                break
            p = sums[(dir, index)]
            if index < n - 2:
                psnr_tmp = compare_psnr(p[12])
                ssim_tmp = my_compare_ssim(p[12])
                psnr_deblur_total.update(psnr_tmp, 1)
                ssim_deblur_total.update(ssim_tmp, 1)
                logger.info("Interp PSNR : " + str(round(psnr_tmp, 4)) + " Interp SSIM : " + str(round(ssim_tmp, 4)))
            if index == 0:
                psnr_tmp = compare_psnr(p[8])
                ssim_tmp = my_compare_ssim(p[8])
                psnr_deblur_total.update(psnr_tmp, 1)
                ssim_deblur_total.update(ssim_tmp, 1)
                logger.info("Interp PSNR : " + str(round(psnr_tmp, 4)) + " Interp SSIM : " + str(round(ssim_tmp, 4)))
            avg_interp_error_abs = np.float64(p[13]["abs"] / p[13]["n"])        # np.mean of exact integers
            interp_error.update(avg_interp_error_abs, 1)
            mse = np.float64(p[13]["sq"] / p[13]["n"])
            if mse == 0:
                return log, summ, True
            PIXEL_MAX = 255.0
            psnr = 20 * math.log10(PIXEL_MAX / math.sqrt(mse))
            ssim_tmp = my_compare_ssim(p[13])
            psnr_interp_total.update(psnr, 1)
            ssim_interp_total.update(ssim_tmp, 1)
            logger.info("deblur error / PSNR : " + str(round(avg_interp_error_abs, 4)) + " / " + str(round(psnr, 4)))
            psnr_tmp = compare_psnr(p[-1])
            ssim_tmp = my_compare_ssim(p[-1])
            psnr_blurry_total.update(psnr_tmp, 1)
            ssim_blurry_total.update(ssim_tmp, 1)
            logger.info("blurry PSNR : " + str(round(psnr_tmp, 4)) + " blurry SSIM : " + str(round(ssim_tmp, 4)) + '\n'
                        + blurry_path(dir, index))
        logger_summary.info("The results for dir:" + dir)
        logger_summary.info("The average interpolation error " + str(round(interp_error.avg, 4)))
        logger_summary.info("Avg. folder" + " blurry psnr " + str(psnr_blurry_total.avg) + " deblur psnr "
                            + str(psnr_interp_total.avg) + " interp psnr " + str(psnr_deblur_total.avg)
                            + " blurry ssim " + str(ssim_blurry_total.avg) + " deblur ssim " + str(ssim_interp_total.avg)
                            + " interp ssim " + str(ssim_deblur_total.avg))
        interp_error_set.update(interp_error.avg, 1)
        psnr_interp_total_set.update(psnr_interp_total.avg, 1)
        ssim_interp_total_set.update(ssim_interp_total.avg, 1)
        psnr_deblur_total_set.update(psnr_deblur_total.avg, 1)
        ssim_deblur_total_set.update(ssim_deblur_total.avg, 1)
        psnr_blurry_total_set.update(psnr_blurry_total.avg, 1)
        ssim_blurry_total_set.update(ssim_blurry_total.avg, 1)
    logger_summary.info("The results for Adobe dataset")
    logger_summary.info("The average interpolation error " + str(round(interp_error_set.avg, 4)))
    logger_summary.info("Avg. testset " + " interp psnr " + str(psnr_deblur_total_set.avg) + " blurry psnr"
                        + str(psnr_blurry_total_set.avg) + " deblur psnr" + str(psnr_interp_total_set.avg)
                        + " interp ssim " + str(ssim_deblur_total_set.avg) + " blurry ssim"
                        + str(ssim_blurry_total_set.avg) + " deblur ssim" + str(ssim_interp_total_set.avg))
    logger_summary.info("runtime per image [s] : %.4f\n" % runtime + "CPU[1] / GPU[0] : 1 \n"
                        + "Extra Data [1] / No Extra Data [0] : 1")
    logger_summary.info(model_size)
    return log, summ, False


def synthetic(folders, seed, zero_at=None):
    """Seeded integer sums and SSIMs per window pair -> (records in test.py's order, the same as dicts)."""
    g = np.random.default_rng(seed)
    recs, sums = [], {}
    for f, n in folders:
        h, w = int(g.integers(7, 40)), int(g.integers(7, 40))
        px = h * w * 3
        for i in range(max(n - 1, 0)):
            rows, d = [], {}
            for k in E._scored(i, n):
                s_abs = int(g.integers(0, 255 * px // 8)) if g.random() > 0.05 else 0
                s_sq = int(g.integers(s_abs, s_abs * 255 + 1)) if s_abs else 0
                if zero_at == (f, i) and k == 13:
                    s_abs = s_sq = 0
                elif k == 13 and s_sq == 0:
                    s_abs, s_sq = 1, 1
                box = float(g.uniform(0.2, 1.0))
                rows.append((float(s_abs), float(s_sq), float(g.uniform(0.2, 1.0)), box))
                d[k] = {"abs": s_abs, "sq": s_sq, "box": box, "n": px}
            recs.append(E.Record(f, i, h, w, tuple(rows)))
            sums[(f, i)] = d
    return recs, sums


FOLDERS = [("a", 2), ("b", 5), ("c", 1), ("d", 9), ("e", 3)]


@pytest.mark.parametrize("seed", range(4))
def test_log_messages_match_test_py(seed):
    recs, sums = synthetic(FOLDERS, seed)
    header = ["In Data: /in ", "Padding mode: 32", "Model path: Joint Model:w.pth", "Save images: /o/60fps_test_results",
              "Flip test: False", "Use ssin method skimage.measure.ssim", "Num. of model parameters is : 123"]
    bp = lambda f, i: f"/in/{f}/{i:05d}.png"   # noqa: E731
    log, summ, stopped = E.test_py_messages(header, FOLDERS, recs, header[-1], 0.25, bp)
    rlog, rsumm, rstop = reference_logs(header, FOLDERS, sums, header[-1], 0.25, bp)
    assert stopped is None and not rstop
    assert log == header + rlog and summ == rsumm
    assert sum(m.startswith("Interp PSNR") for m in log) == sum(max(n - 2, 0) + (n > 1) for _, n in FOLDERS)
    # the records as ranks of world 1 and world 3 gather them: the same text
    for world in (1, 3):
        shards = dist.shard_test_set(dict(FOLDERS), world)
        by_key = {(r.folder, r.i): r for r in recs}
        gathered = [by_key[(f, i)] for pieces in shards for f, rng in pieces for i in rng]
        assert E.test_py_messages(header, FOLDERS, gathered, header[-1], 0.25, bp) == (log, summ, None)


def test_log_stops_where_test_py_returns():
    recs, sums = synthetic(FOLDERS, 7, zero_at=("d", 3))
    bp = lambda f, i: f"/in/{f}/{i:05d}.png"   # noqa: E731
    log, summ, stopped = E.test_py_messages([], FOLDERS, recs, "m", 0.0, bp)
    rlog, rsumm, rstop = reference_logs([], FOLDERS, sums, "m", 0.0, bp)
    assert rstop and stopped == ("d", 3) and (log, summ) == (rlog, rsumm)
    assert not any(m.startswith("The results for Adobe") for m in summ)


def test_batch_metrics_args_are_checked():
    import ctypes as C
    from bin_b200 import _lib
    L = _lib.lib()
    assert L.bin_image_metrics_batch_workspace_bytes(0, 64, 64) == 0
    assert L.bin_image_metrics_batch_workspace_bytes(17, 64, 64) == 0
    assert L.bin_image_metrics_batch_workspace_bytes(3, 64, 64) == 3 * L.bin_image_metrics_workspace_bytes(64, 64)
    p = 1 << 20
    ws = int(L.bin_image_metrics_batch_workspace_bytes(2, 64, 64))
    tab = (C.c_void_p * 2)(p, p)
    nul = (C.c_void_p * 2)(p, None)
    cases = [((tab, tab, 0, 64, 64, 3, 0, p, p, ws), "n must be"),
             ((tab, tab, 17, 64, 64, 3, 0, p, p, ws), "n must be"),
             ((tab, nul, 2, 64, 64, 3, 0, p, p, ws), "null image pointer"),
             ((None, tab, 2, 64, 64, 3, 0, p, p, ws), "null pointer table"),
             ((tab, tab, 2, 64, 64, 1, 1, p, p, ws), "needs c = 3"),
             ((tab, tab, 2, 64, 64, 3, 2, p, p, ws), "unknown flag"),
             ((tab, tab, 2, 6, 64, 3, 0, p, p, ws), "at least 7"),
             ((tab, tab, 2, 64, 64, 3, 0, p + 4, p, ws), "aligned"),
             ((tab, tab, 2, 64, 64, 3, 0, p, p, ws - 1), "workspace too small")]
    for args, msg in cases:
        rc = L.bin_image_metrics_batch_u8(*args, None)
        assert rc != 0 and msg in L.bin_last_error().decode(), (msg, L.bin_last_error())


def test_cli_flag_parsing():
    assert E._flag("True") and E._flag("1") and not E._flag("False") and not E._flag("")
    with pytest.raises(Exception):
        E._flag("maybe")
