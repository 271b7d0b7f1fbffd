"""CPU checks of whole-video streaming (streaming.stream_video): test_py_window against a literal restatement of
test.py's index lists, test_py_names / test_py_writes against a restatement of the files test.py's loop writes, and
the scheduler's plan (VideoPlan) against hand-counted videos and against the properties it must keep for every
length and output selection."""
import itertools

import pytest

from bin_b200 import BinB200Error, streaming as S
from bin_b200.rdn import _window_live

FULL = _window_live(range(14))


def reference_lists(n):
    """test.py:249-258, 334 as written, on positions (test.py scales them by 8 into file numbers right after)."""
    out = []
    frames = list(range(n))
    for index, frame in enumerate(frames):
        if index >= len(frames) - 1:
            break
        first_5_blurry_list = [max(index - 2, 0), max(index - 1, 0), min(index, len(frames) - 1),
                               min(index + 1, len(frames) - 1), min(index + 2, len(frames) - 1)]
        second_5_blurry_list = [max(index - 1, 0), max(index - 0, 0), min(index + 1, len(frames) - 1),
                                min(index + 2, len(frames) - 1), min(index + 3, len(frames) - 1)]
        list_tmp = [first_5_blurry_list[0], first_5_blurry_list[1], first_5_blurry_list[2], first_5_blurry_list[3],
                    first_5_blurry_list[4], second_5_blurry_list[4]]
        out.append(tuple(list_tmp))
    return out


@pytest.mark.parametrize("n", range(1, 16))
def test_window_positions_match_test_py(n):
    assert [S.test_py_window(i, n) for i in range(max(n - 1, 0))] == reference_lists(n)
    for i in (-1, max(n - 1, 0)):
        with pytest.raises(BinB200Error, match="test.py runs windows"):
            S.test_py_window(i, n)


def test_two_frame_video_has_one_window():
    assert S.test_py_window(0, 2) == (0, 0, 0, 1, 1, 1)
    assert reference_lists(2) == [(0, 0, 0, 1, 1, 1)]


def reference_files(n, first):
    """The files test.py:245-299, 380-419 writes, per window in order, into an empty output directory, with time_step
    of length 1 (frame_index 3) and blurry frames named first, first + 8, ... as in the Adobe240 test sets."""
    frames = [str(first + 8 * k).zfill(5) + ".png" for k in range(n)]
    shift_file, offset_file = 1, 0
    exists, out = set(), []
    for index, frame in enumerate(frames):
        if index >= len(frames) - 1:
            break
        second_frame_num = int(int(frame[:-4]) + 8)
        first_gt_deblur = int(int(frame[:-4]) * shift_file + offset_file + 4)
        second_gt_deblur = int(second_frame_num * shift_file + offset_file + 4)
        first_gt_deblur_name = str(first_gt_deblur).zfill(5) + '.png'
        second_gt_deblur_name = str(second_gt_deblur).zfill(5) + '.png'
        interpolated_sharp_list = range(first_gt_deblur + 1, second_gt_deblur)
        middle_frame_name = str(interpolated_sharp_list[3]).zfill(5) + '.png'
        wrote = []
        if middle_frame_name not in exists:
            wrote.append((13, middle_frame_name))
            exists.add(middle_frame_name)
        if index < len(frames) - 2 and second_gt_deblur_name not in exists:
            wrote.append((12, second_gt_deblur_name))
            exists.add(second_gt_deblur_name)
        if first_gt_deblur_name not in exists:
            wrote.append((8, first_gt_deblur_name))
            exists.add(first_gt_deblur_name)
        out.append((int(frame[:-4]), wrote))
    return out


@pytest.mark.parametrize("n", range(1, 12))
@pytest.mark.parametrize("first", [0, 17, 1000])
def test_names_and_writes_match_test_py(n, first):
    got = []
    for i in range(max(n - 1, 0)):
        frame_num = first + 8 * i
        names = S.test_py_names(frame_num)
        got.append((frame_num, [(k, names[k]) for k in S.test_py_writes(i, n)]))
    assert got == reference_files(n, first)


def test_names_of_one_window():
    assert S.test_py_names(8) == {13: "00016.png", 8: "00012.png", 12: "00020.png"}
    assert S.test_py_writes(0, 20) == (13, 12, 8) and S.test_py_writes(5, 20) == (13, 12) and S.test_py_writes(18, 20) == (13,)
    assert S.test_py_writes(0, 2) == (13, 8)


def run_plan(n, live=FULL):
    """[(event, steps)] of one n-frame video: event k = 1..n is the arrival of the k-th frame, "end" the end."""
    plan = S.VideoPlan(live)
    events = [(k + 1, plan.arrive()) for k in range(n)]
    return events + [("end", plan.end())]


def test_plan_of_a_two_frame_video():
    (e1, s1), (e2, s2), (end, last) = run_plan(2)
    assert s1 == [] and s2 == [] and len(last) == 1
    step = last[0]
    assert step.i == 0 and step.frames == (0, 0, 0, 1, 1, 1)
    assert step.fresh == ((0, 0), (0, 1), (1, 1))                # 3 stage-1 calls
    assert step.evict_pairs == ((0, 0), (0, 1), (1, 1)) and step.evict_frames == (0, 1)
    assert step.backbone_calls == 3 + 12 == 13 * 2 - 11


def test_plan_of_a_seven_frame_video():
    """Counted by hand: window i is due at the arrival of frame i+3 (event i+4); windows 4 and 5 at the end."""
    got = [(e, [(s.i, s.frames, s.fresh, s.evict_pairs, s.evict_frames, s.backbone_calls) for s in steps])
           for e, steps in run_plan(7)]
    assert got == [
        (1, []), (2, []), (3, []),
        (4, [(0, (0, 0, 0, 1, 2, 3), ((0, 0), (0, 1), (1, 2), (2, 3)), (), (), 16)]),
        (5, [(1, (0, 0, 1, 2, 3, 4), ((3, 4),), ((0, 0),), (), 13)]),
        (6, [(2, (0, 1, 2, 3, 4, 5), ((4, 5),), ((0, 1),), (0,), 13)]),
        (7, [(3, (1, 2, 3, 4, 5, 6), ((5, 6),), ((1, 2),), (1,), 13)]),
        ("end", [(4, (2, 3, 4, 5, 6, 6), ((6, 6),), ((2, 3),), (2,), 13),
                 (5, (3, 4, 5, 6, 6, 6), (), ((3, 4), (4, 5), (5, 6), (6, 6)), (3, 4, 5, 6), 12)]),
    ]
    steps = [s for _, ss in run_plan(7) for s in ss]
    assert len(steps) == 6 and sum(len(s.fresh) for s in steps) == 8
    assert sum(s.backbone_calls for s in steps) == 13 * 7 - 11 == 80


def test_plan_of_a_three_frame_video():
    steps = run_plan(3)
    assert all(s == [] for _, s in steps[:-1])
    w0, w1 = steps[-1][1]
    assert (w0.frames, w0.fresh, w0.evict_pairs) == ((0, 0, 0, 1, 2, 2), ((0, 0), (0, 1), (1, 2), (2, 2)), ())
    assert (w1.frames, w1.fresh, w1.evict_frames) == ((0, 0, 1, 2, 2, 2), (), (0, 1, 2))
    assert w0.backbone_calls + w1.backbone_calls == 13 * 3 - 11


def test_plan_of_a_selection():
    """(13, 8, 12): stage-1 position 0 is dead, 9 calls of stages 2-4 per window.  Every pair at position 0 of a window
    is at position 1 of the same or the window before, so every pair is still evaluated once: 8 + 6 * 9."""
    steps = [s for _, ss in run_plan(7, _window_live((13, 8, 12))) for s in ss]
    assert [s.fresh for s in steps] == [((0, 0), (0, 1), (1, 2), (2, 3)), ((3, 4),), ((4, 5),), ((5, 6),), ((6, 6),), ()]
    assert [s.backbone_calls for s in steps] == [13, 10, 10, 10, 10, 9]


@pytest.mark.parametrize("wanted", [range(14), (13, 8, 12), (9,), (0,), (10,), (4, 11)], ids=str)
def test_plan_keeps_its_promises(wanted):
    """For every length up to 30: windows 0..N-2 in order, each due as soon as its frames have arrived; every live pair
    of a window is held or fresh and evaluated once per video; what is dropped is read by no later window; at most six
    frames and five pairs are held; the call count is the distinct live pairs plus the stages 2-4 of every window."""
    live = _window_live(wanted)
    live1 = [a for a in range(5) if (1, a) in live]
    later = sum(1 for n in live if n[0] in (2, 3, 4))
    for n in range(0, 31):
        windows = [S.test_py_window(i, n) for i in range(max(n - 1, 0))]
        reads = [{(w[a], w[a + 1]) for a in live1} for w in windows]
        held_frames, held_pairs, seen, order = set(), set(), set(), []
        for event, steps in run_plan(n, live):
            if event != "end":
                held_frames.add(event - 1)
            for s in steps:
                order.append(s.i)
                assert s.frames == windows[s.i]
                assert max(s.frames) < (n if event == "end" else event)     # its frames have arrived
                if event == "end":
                    assert s.i >= n - 3                                       # no frame i+3: it could not run earlier
                else:
                    assert s.frames[5] == event - 1 == s.i + 3                # due at the arrival of frame i+3
                assert set(s.frames) <= held_frames and len(held_frames) <= 6
                assert not set(s.fresh) & seen and reads[s.i] <= held_pairs | set(s.fresh)
                seen |= set(s.fresh)
                held_pairs |= set(s.fresh)
                assert len(held_pairs) <= 5
                assert set(s.evict_pairs) <= held_pairs and set(s.evict_frames) <= held_frames
                for j in range(s.i + 1, n - 1):
                    assert not set(s.evict_pairs) & reads[j] and not set(s.evict_frames) & set(windows[j])
                held_pairs -= set(s.evict_pairs)
                held_frames -= set(s.evict_frames)
                assert s.backbone_calls == len(s.fresh) + later
        assert order == list(range(max(n - 1, 0)))
        assert not held_pairs and (n < 2 or not held_frames)
        assert seen == set().union(*reads)
        if wanted == range(14) and n >= 2:
            assert len(seen) == n + 1 and len(seen) + later * (n - 1) == 13 * n - 11


def test_plan_of_the_benchmarked_video():
    """The 20-frame video of tools/bench_video.py: 249 backbone calls against 17 * 19 = 323 per window."""
    steps = list(itertools.chain.from_iterable(s for _, s in run_plan(20)))
    assert len(steps) == 19 and sum(s.backbone_calls for s in steps) == 249 == 13 * 20 - 11
    assert 17 * len(steps) == 323
