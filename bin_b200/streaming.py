"""Sliding-window inference over a video (the caller loop of test.py:222-402), SURVEY 8f ranks 1-2.

test.py slides the 6-frame window by one blurry frame: window k uses frames i..i+5, window k+1 uses i+1..i+6.
Four of the five stage-1 backbone calls of window k+1 (adjacent frame pairs) were already evaluated for window k --
they are pure functions of two frames and the stage-1 weights -- so a stream needs 13 backbone calls per window
instead of the 17 unique ones (20 in the reference).  Every frame is uploaded once (as uint8) instead of six times.
Stages 2-4 are NOT reusable: window k's step 1 used LSTM history where window k+1's step 0 duplicates its first
input (RDN.py:375-389), so they are recomputed; the outputs are bit-identical to calling the module per window.

stream_video walks a whole video in test.py's order (test.py:249-258, 334), the clamped windows at both ends included;
StreamingBIN returns only the windows of six distinct frames.
"""
from __future__ import annotations

from collections import OrderedDict
from typing import Dict, Iterable, List, NamedTuple, Optional, Tuple

import torch

from . import ops
from ._lib import BinB200Error, check, lib
from .rdn import (_OUT_NODE, _ensemble_of, _flipx4_mean_at, _outputs_of, _prec_of, _selected, _window_fwd,
                  _window_live)


def test_py_padding(h: int, w: int) -> Tuple[int, int, int, int]:
    """(left, right, top, bottom) exactly as test.py:348-364 / demo.py."""
    if w != ((w >> 7) << 7):
        wp = ((w >> 7) + 1) << 7
        pl = int((wp - w) / 2)
        pr = wp - w - pl
    else:
        pl = pr = 32
    if h != ((h >> 7) << 7):
        hp = ((h >> 7) + 1) << 7
        pt = int((hp - h) / 2)
        pb = hp - h - pt
    else:
        pt = pb = 32
    return pl, pr, pt, pb


def upload_frame_u8(img_u8: torch.Tensor, pad: Tuple[int, int, int, int], device) -> torch.Tensor:
    """uint8 HWC BGR image (what cv2.imread returns; host or device) -> (1,3,Hp,Wp) fp32 RGB [0,1] on `device`,
    replicate-padded: read_image (test.py:44-56) + ReplicationPad2d (test.py:366-371) in one kernel."""
    if img_u8.dtype != torch.uint8 or img_u8.dim() != 3 or img_u8.shape[2] != 3:
        raise BinB200Error("upload_frame_u8 expects a uint8 HWC (h,w,3) BGR image")
    h, w, _ = img_u8.shape
    pl, pr, pt, pb = pad
    dev = torch.device(device)
    with torch.cuda.device(dev):
        d = img_u8.contiguous().to(dev, non_blocking=True)
        out = torch.empty((1, 3, h + pt + pb, w + pl + pr), dtype=torch.float32, device=dev)
        check(lib().bin_u8_to_frame(d.data_ptr(), h, w, pl, pr, pt, pb, out.data_ptr(), ops._stream()))
    return out


def tensor2img_u8(t: torch.Tensor, crop: Optional[Tuple[int, int, int, int]] = None) -> torch.Tensor:
    """(1,3,H,W) / (3,H,W) fp32 RGB -> uint8 HWC BGR on the device (utils/util.py:113-137), optional (top,left,h,w) crop."""
    x = t.reshape(-1, t.shape[-2], t.shape[-1])
    if x.shape[0] != 3 or not x.is_cuda or x.dtype != torch.float32:
        raise BinB200Error("tensor2img_u8 expects one fp32 CUDA image with 3 channels")
    x = x.contiguous()
    Hs, Ws = x.shape[-2:]
    top, left, h, w = crop if crop is not None else (0, 0, Hs, Ws)
    with torch.cuda.device(x.device):
        out = torch.empty((h, w, 3), dtype=torch.uint8, device=x.device)
        check(lib().bin_tensor2img_u8(x.data_ptr(), Hs, Ws, top, left, h, w, out.data_ptr(), ops._stream()))
    return out


class StreamingBIN:
    """Feed frames one at a time; from the 6th frame on, every push returns the 14-tuple of that window.

    With the net's x4 flip self-ensemble on (rdn.set_self_ensemble), every pushed frame is expanded once into its four
    orientations (4B items), the stage-1 cache holds 4B outputs, and each window's 14 outputs are flipped back and
    averaged: the same bits as calling the net per window.

    With an output selection on the net (rdn.set_outputs) a window runs only the backbone calls its wanted outputs depend
    on, and returns what the net would: for (13, 8, 12) the pair of the two oldest frames is never evaluated, so the
    first window costs 13 calls and every later one 10.

    It returns only the windows of six distinct frames; stream_video walks a whole video in test.py's order, the
    clamped windows at both ends included."""

    def __init__(self, net):
        self.net = net
        self.frames: List[Tuple[int, torch.Tensor]] = []            # (frame id, (B,3,H,W) or expanded (4B,3,H,W) tensor)
        self.s1: "OrderedDict[Tuple[int, int], torch.Tensor]" = OrderedDict()   # stage-1 output per adjacent frame pair
        self.next_id = 0
        self.backbone_calls = 0
        self.key = None                                # (ensemble mode, output selection, frame shape) of the cache

    def reset(self):
        self.frames.clear()
        self.s1.clear()

    @torch.no_grad()
    def push(self, frame: torch.Tensor):
        if not frame.is_cuda or frame.dtype != torch.float32 or frame.dim() != 4 or frame.shape[1] != 3:
            raise BinB200Error("StreamingBIN.push expects a (B,3,H,W) fp32 CUDA frame (see upload_frame_u8)")
        ensemble = _ensemble_of(self.net)
        key = (ensemble, _outputs_of(self.net), frame.shape)
        if self.frames and self.key != key:
            self.reset()
        self.key = key
        frame = frame.contiguous()
        if ensemble is not None:
            with torch.cuda.device(frame.device):
                frame = ops.flipx4_expand([frame])[0]
        self.frames.append((self.next_id, frame))
        self.next_id += 1
        if len(self.frames) > 6:
            old = self.frames.pop(0)[0]
            for key in [k for k in self.s1 if old in k]:
                del self.s1[key]
        if len(self.frames) < 6:
            return None
        return self._window()

    def _window(self):
        ids = [i for i, _ in self.frames]
        o, calls = _cached_window(self.net, [f for _, f in self.frames], [(ids[a], ids[a + 1]) for a in range(5)],
                                  self.s1, *self.key[:2])
        self.backbone_calls += calls
        return o


def _later_calls(live) -> int:
    """Backbone calls of stages 2-4 among the window nodes `live`: every window runs them anew."""
    return sum(1 for n in live if n[0] in (2, 3, 4))


def _cached_window(net, F, pairs, cache, ensemble, sel):
    """One window on the six frames F in the net's modes (ensemble: F are expanded; sel: the net's output selection)
    -> (what the net returns for it, the backbone calls run).  pairs names the frame pair of each stage-1 position.
    Stage 1 runs only the live pairs `cache` does not hold, each distinct pair once, and adds them to it."""
    wanted = range(14) if sel is None else sel[0]
    live = _window_live(wanted)
    s1 = [cache.get(p) for p in pairs]
    fresh = {pairs[a] for a in range(5) if (1, a) in live and s1[a] is None}
    o = _window_fwd(net, F, live, s1, keys=pairs)
    for i, n in enumerate(_OUT_NODE):
        if n[0] == 1 and o[i] is not None:
            cache[pairs[n[1]]] = o[i]
    if ensemble is not None:
        o = tuple(_flipx4_mean_at(o, wanted))
    return (o if sel is None else _selected(o, sel)), len(fresh) + _later_calls(live)


def test_py_window(i: int, n: int) -> Tuple[int, ...]:
    """The positions of the six frames that window i of an n-frame video reads in test.py: the five of
    first_5_blurry_list, then the last of second_5_blurry_list (test.py:257-258, 334), clamped to the video, so the
    first two windows and the last two repeat an end frame.  test.py runs the windows i = 0 .. n-2 (test.py:249-255):
    a video of fewer than two frames has none, and one of two frames has the single window (0, 0, 0, 1, 1, 1)."""
    if not 0 <= i <= n - 2:
        raise BinB200Error(f"test.py runs windows 0..{n - 2} of a {n}-frame video; there is no window {i}")
    return max(i - 2, 0), max(i - 1, 0), min(i, n - 1), min(i + 1, n - 1), min(i + 2, n - 1), min(i + 3, n - 1)


def test_py_names(frame_num: int) -> Dict[int, str]:
    """The files test.py writes for the window whose blurry frame is named frame_num (test.py:287-299, 380-419), by
    output index: the interpolated frame Ft_p[13] at frame_num + 8, the first deblurred frame Ft_p[8] at frame_num + 4
    and the second deblurred frame Ft_p[12] at frame_num + 12.  test_py_writes says which of them a window writes."""
    return {k: str(frame_num + d).zfill(5) + ".png" for k, d in ((13, 8), (8, 4), (12, 12))}


def test_py_writes(i: int, n: int) -> Tuple[int, ...]:
    """The outputs that window i of an n-frame video writes in test.py, in its order (test.py:380-419), into an output
    directory that starts empty: Ft_p[13] always; Ft_p[12] while i < n - 2 (test.py:404); Ft_p[8] only in window 0.
    test.py writes a file only if it is not there yet, and from window 1 on the first deblurred frame is the file the
    window before wrote as its second: the blurry frames are named 8 apart, as test.py assumes when it names its
    inputs (test.py:262-263)."""
    test_py_window(i, n)
    return (13,) + ((12,) if i < n - 2 else ()) + ((8,) if i == 0 else ())


class WindowStep(NamedTuple):
    """One window of VideoPlan: what stream_video runs and what it drops after it."""
    i: int                                          # window index, 0 .. N-2
    frames: Tuple[int, ...]                         # the six frame positions it reads (test_py_window)
    fresh: Tuple[Tuple[int, int], ...]              # live stage-1 pairs (frame positions) no earlier window evaluated
    evict_pairs: Tuple[Tuple[int, int], ...]        # stage-1 outputs no later window reads
    evict_frames: Tuple[int, ...]                   # frames no later window reads
    backbone_calls: int                             # len(fresh) + the live calls of stages 2-4


class VideoPlan:
    """stream_video's schedule, without tensors: call arrive() once per frame and end() when the frames end; each
    returns the windows (WindowStep) due at that point, in order.  Window i is due once frame min(i+3, N-1) has arrived;
    without n the last two windows read no frame i+3 and are due at the end.  live is the window's node set
    (rdn._window_live).

    windows = range(a, b) plans only windows a .. b-1 of the video, from frames that start at position max(a-2, 0)
    (next_pos names the position the next frame takes); n, the video's frame count, is needed only when window b-1 reads
    a clamped end frame (b-1 >= n-3), and end() raises when it was needed and not given.  complete says that every
    window of the range is out, so no more frames need to arrive.

    A stage-1 output is named by its pair of frame positions and evaluated once, the first time a window of the plan
    reads it at a live position (so the first window of a range evaluates all its live pairs).  Later windows never read
    below the first pair (and first frame) of the next window, so after window i everything below window i+1's is
    dropped: at most six frames and five pairs are held.  With all 14 outputs an N-frame video costs N+1 stage-1 calls,
    12 per window for stages 2-4, 13N - 11 in all; a range of windows that reads no clamped frame b-a+4 stage-1 calls
    and 12 (b-a) for stages 2-4."""

    def __init__(self, live, windows: Optional[range] = None, n: Optional[int] = None):
        if windows is not None and (not isinstance(windows, range) or windows.step != 1 or not 0 <= windows.start < windows.stop):
            raise BinB200Error(f"windows must be a non-empty range(a, b) with 0 <= a < b; got {windows!r}")
        if n is not None and windows is not None and windows.stop > n - 1:
            raise BinB200Error(f"an {n}-frame video has windows 0..{n - 2}; {windows!r} is not among them")
        self.live1 = [a for a in range(5) if (1, a) in live]
        self.later = _later_calls(live)
        self.n = n
        self.first = 0 if windows is None else windows.start
        self.stop = None if windows is None else windows.stop          # None: to the end of the video
        if self.stop is None and n is not None:
            self.stop = max(n - 1, 0)
        self.start = max(self.first - 2, 0)         # position of the first frame
        self.arrived = 0
        self.ended = False
        self.done = self.first                      # the next window to return
        self.pairs: set = set()                     # pairs evaluated and not dropped
        self.low = self.start                       # the lowest frame position not dropped

    @property
    def next_pos(self) -> int:
        return self.start + self.arrived

    @property
    def complete(self) -> bool:
        return self.stop is not None and self.done >= self.stop

    def arrive(self) -> List[WindowStep]:
        if self.complete or (self.n is not None and self.next_pos >= self.n):
            raise BinB200Error(f"VideoPlan: frame {self.next_pos} arrived after the plan's last window")
        self.arrived += 1
        stop = self.next_pos - 3
        if self.n is not None and self.next_pos == self.n:
            stop = self.stop                        # the last frame: the clamped windows are due
        return self._due(stop if self.stop is None else min(stop, self.stop))

    def end(self) -> List[WindowStep]:
        self.ended = True
        n = self.next_pos
        if self.stop is None:
            return self._due(n - 1)
        if self.complete:
            return []
        if self.n is not None:
            raise BinB200Error(f"the frames ended at position {n - 1}; windows up to {self.stop - 1} of the "
                               f"{self.n}-frame video need frames up to {min(self.stop + 2, self.n - 1)}")
        raise BinB200Error(f"the frames ended at position {n - 1} before window {self.done} was due: windows "
                           f"{self.done}..{self.stop - 1} read clamped end frames, so the video's length n is needed")

    def _n(self) -> int:
        """The frame count windows are clamped to: n, or while it is unknown the frames so far (no window due before
        the end of an unknown-length video reads a clamped end frame)."""
        return self.n if self.n is not None else self.next_pos

    def _due(self, stop: int) -> List[WindowStep]:
        steps, n = [], self._n()
        last = self.stop - 1 if self.stop is not None else (n - 2 if self.ended else None)
        for i in range(self.done, stop):
            pos = test_py_window(i, n)
            pairs = [(pos[a], pos[a + 1]) for a in self.live1]
            fresh = tuple(dict.fromkeys(p for p in pairs if p not in self.pairs))
            self.pairs.update(fresh)
            if i == last:
                first, low = (n, n), self.next_pos  # the plan's last window: drop everything
            else:
                nxt = test_py_window(i + 1, n)
                first, low = (nxt[0], nxt[1]), nxt[0]
            gone = tuple(sorted(p for p in self.pairs if p < first))
            self.pairs.difference_update(gone)
            steps.append(WindowStep(i, pos, fresh, gone, tuple(range(self.low, low)), len(fresh) + self.later))
            self.low = low
        self.done = max(self.done, stop)
        return steps


class VideoStream:
    """The iterator stream_video returns: (i, outputs) per window; backbone_calls counts the calls run so far."""

    def __init__(self, net, frames: Iterable[torch.Tensor], windows: Optional[range] = None, n: Optional[int] = None):
        self.net = net
        self.backbone_calls = 0
        self._range = (windows, n)
        VideoPlan(frozenset(), windows, n)          # reject a bad range now rather than at the first frame
        self._it = self._windows(iter(frames))

    def __iter__(self) -> "VideoStream":
        return self

    def __next__(self):
        return next(self._it)

    def _windows(self, frames):
        held: Dict[int, torch.Tensor] = {}          # frame position -> (B,3,H,W), or (4B,3,H,W) expanded
        cache: Dict[Tuple[int, int], torch.Tensor] = {}     # frame-position pair -> stage-1 output
        plan = mode = shape = None
        for frame in frames:
            if not (isinstance(frame, torch.Tensor) and frame.is_cuda and frame.dtype == torch.float32
                    and frame.dim() == 4 and frame.shape[1] == 3):
                raise BinB200Error("stream_video expects (B,3,H,W) fp32 CUDA frames (see upload_frame_u8)")
            if plan is None:
                mode, shape = self._mode(), (frame.shape, frame.device)
                plan = VideoPlan(_window_live(range(14) if mode[1] is None else mode[1][0]), *self._range)
            elif (frame.shape, frame.device) != shape:
                raise BinB200Error(f"stream_video: frame {plan.arrived} is {tuple(frame.shape)} on {frame.device}; "
                                   f"the video's first frame is {tuple(shape[0])} on {shape[1]}")
            frame = frame.contiguous()
            if mode[0] is not None:
                with torch.no_grad(), torch.cuda.device(frame.device):
                    frame = ops.flipx4_expand([frame])[0]
            held[plan.next_pos] = frame
            del frame                               # held[] alone keeps it, until the plan drops it
            for step in plan.arrive():
                yield self._run(step, held, cache, mode)
            if plan.complete:
                return                              # the range is out: read no further frame
        if plan is None:
            plan = VideoPlan(frozenset(), *self._range)
        for step in plan.end():
            yield self._run(step, held, cache, mode)

    def _mode(self):
        return _ensemble_of(self.net), _outputs_of(self.net), _prec_of(self.net)

    @torch.no_grad()
    def _run(self, step: WindowStep, held, cache, mode):
        if self._mode() != mode:
            raise BinB200Error("stream_video: the net's self-ensemble, output selection or precision changed during "
                               "the video; start a new stream_video after changing them")
        pairs = [(step.frames[a], step.frames[a + 1]) for a in range(5)]
        o, calls = _cached_window(self.net, [held[p] for p in step.frames], pairs, cache, *mode[:2])
        self.backbone_calls += calls
        for p in step.evict_pairs:
            cache.pop(p, None)
        for p in step.evict_frames:
            del held[p]
        return step.i, o


def stream_video(net, frames: Iterable[torch.Tensor], windows: Optional[range] = None,
                 n: Optional[int] = None) -> VideoStream:
    """Every window test.py runs over a video, in its order: for frames F[0..N-1] (an iterable of (B,3,H,W) fp32 CUDA
    frames, e.g. from upload_frame_u8), yields (i, outputs) for i = 0 .. N-2, where outputs is exactly what
    net(*[F[j] for j in test_py_window(i, N)]) returns, in the net's precision, output selection and self-ensemble
    modes (read when the first frame arrives; changing one during the video raises).  N need not be known: window i is
    yielded once frame i+3 has arrived, and the last two windows when the iterable ends.

    A stage-1 output is kept while a later window can still read it and evaluated once per video, so with all 14
    outputs a video costs 13N - 11 backbone calls where calling the net per window costs 17(N-1) (VideoPlan); the
    iterator's backbone_calls counts them.  At most six frames (expanded once each under the ensemble) and the stage-1
    outputs a later window reads are held.  Outputs at positions 0-3 and 10 are those stage-1 tensors, shared with other
    windows (and, in the first and the last window, between two positions of one tuple): read them, do not write them.  Inference
    only: like StreamingBIN.push, every window runs under torch.no_grad().

    windows = range(a, b) runs only windows a .. b-1 (a piece of the video, e.g. one rank's share): `frames` then starts
    at position max(a-2, 0), and no frame after position min(b+2, N-1) is read.  n = N is needed only when a window of
    the range reads a clamped end frame (b-1 >= N-3); without it that raises when the frames end.  The first window of
    a range evaluates all its live stage-1 pairs, so a range costs at most 4 stage-1 calls more than the same windows
    inside a whole-video stream."""
    return VideoStream(net, frames, windows, n)
