"""demo.py's blurry-video conversion (demo.py:64-324) on one or more GPUs: a folder of blurry 30 fps frames in, deblurred
and interpolated frames out.

run_demo runs the windows demo.py runs, in its order, over every folder of input_path and writes the files demo.py
writes, through the loop evaluate_testset uses (evaluate.window_loop):

  * windows are streamed per video (streaming.stream_video), each frame decoded once, on host threads that read ahead;
  * Ft_p[13], Ft_p[8] and Ft_p[12] (rdn.set_outputs) are cropped on the device (tensor2img_u8) and encoded by the GPU
    PNG encoder (png.encode_png_async); a host thread writes the files;
  * with several ranks, each runs a contiguous run of windows (dist.shard_test_set) and writes its own files.

What demo.py does, and where:

  * the folders are sorted(os.listdir(input_path)) (demo.py:136), written to output_path/<folder>/ (demo.py:104-108,
    170-171): no 60fps_test_results/<netName> level as in test.py;
  * window i = 0 .. N-2 of an N-frame folder reads streaming.test_py_window(i, N), the inputs named first + 8 * position
    (demo.py:179-205, 248), padded as streaming.test_py_padding (demo.py:262-280);
  * the names come from the listed name `frame` of window i (demo.py:210-222): Ft_p[8] to frame + 4, Ft_p[12] to
    frame + 12 while i < N - 2 (demo.py:318), the interpolated Ft_p[13] to frame + 5 + j (interpolated_sharp_list[j]);
    each file is written only if it is not there yet (demo.py:290, 319, 323), so in a fresh directory only window 0
    writes Ft_p[8]: every later window's frame + 4 is the window before's frame + 12;
  * N_frames = round(1 / time_step) (demo.py:101): j = 3 alone when N_frames == 2 (demo.py:226-231), the image at
    frame + 8; otherwise j runs over zip(range(N_frames - 1), range(7)) (demo.py:153, 234, 237): 0..6 for 0.125,
    0..2 for 0.25, none for N_frames <= 1.  Both deblurred writes sit inside that loop, so with no j nothing is
    written (and nothing is run here);
  * the net has no time input: frame_index is appended to testData (demo.py:286) and test_set_input drops it
    (bin_model.py:260), so every j of a window is the same Ft_p[13] image under another name.  It is encoded once and
    the same bytes are written under each name, where demo.py runs the window once per j;
  * the yml is read for network_G and path (demo.py:82, 92, 156-161): which_model_G bin_stage4, nframes 6 (which forces
    version 1, demo.py:158-161), and the weights path.pretrain_model_G loaded with path.strict_load
    (bin_model.py:602-606);
  * the messages: "We interp the 30 fps blurry video to ... fps slow-motion video!" (demo.py:111), "In Data",
    "Padding mode", "Model path" and "Save images" (demo.py:139-142), and "interpolate middle frame" or "interpolate all
    7 frames" (demo.py:227, 235).

Where this departs from demo.py:

  * an output directory that already holds a file the run would write raises before anything runs: demo.py skips the
    window when its interpolated file exists, then writes the deblurred images left from an earlier iteration
    (demo.py:290-324), so a partly written directory is not resumed;
  * the blurry frames of a folder must be named first, first + 8, ...: demo.py names its inputs that way (demo.py:196-205)
    but its outputs from the listing, and only such folders give one answer;
  * the 1280x720 assert (demo.py:259-260) is not imposed;
  * demo.py skips a window whose first input does not have 3 channels (demo.py:256-257); cv2.imread returns 3 channels,
    so that never happens, and frames are decoded in colour the same way here without the check;
  * "interpolate ..." is printed once rather than per window, and one closing line of windows/s and seconds per window
    replaces the per-image time lines (demo.py:304);
  * a time_step <= 0 is refused (demo.py divides by it), and so is a yml without pretrain_model_G when no --weights is
    given (demo.py would run untrained weights).

python -m bin_b200.demo takes demo.py's arguments (see main()); under torchrun it shards over the ranks."""
from __future__ import annotations

import argparse
import os
from typing import Dict, List, NamedTuple, Optional, Tuple

import torch

from . import dist as bdist
from . import rdn
from ._lib import BinB200Error
from .evaluate import _flag, _gather, folder_info, load_weights, window_loop, window_nets
from .streaming import test_py_window

WANTED = (13, 8, 12)                    # the three outputs demo.py writes (demo.py:294-296)
VAL_FPS = 30                            # demo.py:99
PAD = 32                                # demo.py:114, printed as the padding mode
WHO = "run_demo"


# ----------------------------------------------------------------------------- names (demo.py:164-324)
def demo_py_steps(time_step: float) -> Tuple[int, ...]:
    """The j demo.py runs per window for time_step (demo.py:101, 153, 226-237): each names interpolated_sharp_list[j]."""
    if not time_step > 0:
        raise BinB200Error(f"time_step must be > 0, got {time_step!r}")
    n_frames = round(1 / time_step)
    if n_frames == 2:
        return (3,)
    return tuple(j for _, j in zip(range(n_frames - 1), range(7)))


def demo_py_writes(i: int, n: int, time_step: float, first: int = 0) -> Dict[int, List[str]]:
    """The files window i of an n-frame folder writes in demo.py into an output directory that starts empty, by output
    index (demo.py:290-324): Ft_p[13] under frame + 5 + j for each j of demo_py_steps, Ft_p[12]
    under frame + 12 while i < n - 2, Ft_p[8] under frame + 4 in window 0 only; frame = first + 8 i is the window's
    blurry frame (the names run 8 apart, so from window 1 on frame + 4 is the file the window before wrote as its
    frame + 12).  No j: nothing."""
    test_py_window(i, n)
    steps = demo_py_steps(time_step)
    if not steps:
        return {}
    frame = first + 8 * i
    name = lambda num: str(num).zfill(5) + ".png"   # noqa: E731
    out = {13: [name(frame + 5 + j) for j in steps]}
    if i < n - 2:
        out[12] = [name(frame + 12)]
    if i == 0:
        out[8] = [name(frame + 4)]
    return out


def demo_py_messages(input_path: str, output_path: str, time_step: float, model_path: str) -> List[str]:
    """demo.py's header (demo.py:111, 139-142) and its window message (demo.py:227, 235)."""
    return ["We interp the " + str(VAL_FPS) + " fps blurry video to " + str(round(1 / time_step) * VAL_FPS)
            + " fps slow-motion video!",
            'In Data: {} '.format(input_path), 'Padding mode: {}'.format(PAD),
            'Model path: {}'.format("Joint Model:" + model_path), 'Save images: {}'.format(output_path),
            "interpolate middle frame" if round(1 / time_step) == 2 else "interpolate all 7 frames"]


# ----------------------------------------------------------------------------- the run
class DemoStats(NamedTuple):
    windows: int                        # windows run, over all ranks
    files: int                          # files written, over all ranks
    seconds: float                      # seconds of the window loops, summed over the ranks
    wall: float                         # the slowest rank's seconds


def run_demo(net, input_path: str, output_path: str, *, time_step: float = 0.5, rank: Optional[int] = None,
             world: Optional[int] = None, decode_threads: int = 8, model_path: str = "", verbose: bool = True) -> DemoStats:
    """demo.py's conversion (demo.py:64-324): the blurry frames under input_path/<folder>/ (named 8 apart), the images
    written to output_path/<folder>/ under demo_py_writes' names.  net: a BIN window net, or a module holding one, on
    the device it runs on; it computes only (13, 8, 12) during the call, in its precision, self-ensemble and backbone,
    and its output selection is restored afterwards.  With verbose, rank 0 prints demo.py's messages ("Model path:
    Joint Model:<model_path>") and a closing line of windows/s and seconds per window.

    rank / world default to the initialised process group, else (0, 1).  Each rank runs its contiguous run of windows
    (dist.shard_test_set) and writes its files; the ranks meet once at the end, to sum the counts.  Raises BinB200Error,
    before any window runs, if a file it would write exists."""
    if rank is None or world is None:
        if torch.distributed.is_available() and torch.distributed.is_initialized():
            rank, world = torch.distributed.get_rank(), torch.distributed.get_world_size()
        else:
            rank, world = 0, 1
    if not 0 <= rank < world:
        raise BinB200Error(f"{WHO}: rank {rank} is not in 0..{world - 1}")
    steps = demo_py_steps(time_step)
    nets = window_nets(net, WHO)
    dev = next(net.parameters()).device
    subdir = sorted(os.listdir(input_path))                                      # demo.py:136
    info = {f: folder_info(input_path, f, WHO) for f in subdir}
    pieces = bdist.shard_test_set({f: info[f][0] for f in subdir}, world)[rank] if steps else []

    def outputs(folder, i, n):
        return {k: [os.path.join(output_path, folder, f) for f in names]
                for k, names in demo_py_writes(i, n, time_step, info[folder][1]).items()}

    files = [p for folder, rng in pieces for i in rng for ps in outputs(folder, i, info[folder][0]).values() for p in ps]
    for p in files:
        if os.path.exists(p):
            raise BinB200Error(f"{WHO}: {p} exists; demo.py would skip that window and write other images, so convert "
                               "into a directory without its images")
    if verbose and rank == 0:
        for msg in demo_py_messages(input_path, output_path, time_step, model_path):
            print(msg)
    for f in subdir:
        os.makedirs(os.path.join(output_path, f), exist_ok=True)               # demo.py:106-107, 170-171

    seconds = 0.0
    if pieces:
        def frame_path(folder, pos):
            return os.path.join(input_path, folder, str(info[folder][1] + 8 * pos).zfill(5) + ".png")

        saved = [getattr(m, "outputs", None) for m in nets]
        for m in nets:
            rdn.set_outputs(m, WANTED)
        try:
            seconds = window_loop(nets[0], dev, pieces, info, frame_path, outputs, threads=decode_threads, who=WHO)
        finally:
            for m, sel in zip(nets, saved):
                m.outputs = sel
    ranks = _gather((sum(len(r) for _, r in pieces), len(files), seconds), world)
    stats = DemoStats(sum(r[0] for r in ranks), sum(r[1] for r in ranks), sum(r[2] for r in ranks),
                      max(r[2] for r in ranks))
    if verbose and rank == 0:
        print(closing_line(stats, world))
    return stats


def closing_line(stats: DemoStats, world: int) -> str:
    if not stats.windows:
        return "no window run: this time_step writes no image"
    rate = stats.windows / stats.wall if stats.wall > 0 else float("inf")
    return (f"{stats.windows} windows, {stats.files} images on {world} GPU(s) in {stats.wall:.3f} s: {rate:.2f} "
            f"windows/s, {stats.seconds / stats.windows:.4f} s per window (summed over the ranks)")


# ----------------------------------------------------------------------------- command line
class DemoOptions(NamedTuple):
    pretrain_model_G: Optional[str]
    strict_load: bool


def parse_options(opt: dict) -> DemoOptions:
    """The keys of a yml demo.py reads (option.parse(opt, is_train=False), demo.py:82-92, 156-161).  Raises
    BinB200Error naming the key for a model this driver does not run: which_model_G other than bin_stage4, nframes
    other than 6."""
    g = opt.get("network_G") if isinstance(opt, dict) else None
    g = g if isinstance(g, dict) else {}
    if g.get("which_model_G") != "bin_stage4":
        raise BinB200Error(f"network_G.which_model_G: {g.get('which_model_G')!r} is not run here; only bin_stage4 is")
    if g.get("nframes") is None or int(g["nframes"]) != 6:
        raise BinB200Error(f"network_G.nframes: {g.get('nframes')!r}; only 6 (the 14-output bin_stage4 window, "
                           "version 1) is run here")
    path = opt.get("path") or {}
    p = path.get("pretrain_model_G")
    return DemoOptions(None if p in (None, "") else os.path.expanduser(str(p)), bool(path.get("strict_load", True)))


def load_options(path: str) -> DemoOptions:
    import yaml
    with open(path) as fh:
        return parse_options(yaml.safe_load(fh))


def _arch(v: str) -> Tuple[int, int]:
    try:
        g0, d = (int(x) for x in v.split(","))
    except ValueError:
        raise argparse.ArgumentTypeError(f"--arch takes G0,D (e.g. 64,6), got {v!r}") from None
    return g0, d


def parse_args(argv=None) -> argparse.Namespace:
    ap = argparse.ArgumentParser(description="demo.py's blurry-video conversion on the GPU (one process per GPU under "
                                             "torchrun)")
    ap.add_argument("--netName", required=True)
    ap.add_argument("--input_path", required=True)
    ap.add_argument("--output_path", required=True)
    ap.add_argument("--time_step", type=float, default=0.5)
    ap.add_argument("--gpu_id", default=None, help="CUDA_VISIBLE_DEVICES for a run outside torchrun")
    ap.add_argument("--opt", required=True, help="the option yml, e.g. options/train/train_adobe_stage4.yml")
    ap.add_argument("--direct_interp", type=_flag, nargs="?", const=True, default=False,
                    help="accepted and unused, as in demo.py")
    ap.add_argument("--launcher", choices=("none", "pytorch"), default="none",
                    help="accepted; torchrun's environment decides")
    ap.add_argument("--local_rank", type=int, default=0, help="accepted; LOCAL_RANK decides")
    ap.add_argument("--weights", default=None, help="a bin_stage4 checkpoint in place of path.pretrain_model_G")
    ap.add_argument("--precision", choices=("fp16", "fp32"), default="fp16")
    ap.add_argument("--flipx4", action="store_true", help="x4 flip self-ensemble")
    ap.add_argument("--arch", type=_arch, default=None, help="backbone G0,D of a light window, e.g. 64,6")
    ap.add_argument("--decode_threads", type=int, default=8)
    return ap.parse_args(argv)


def weights_of(args: argparse.Namespace, opts: DemoOptions) -> Tuple[str, bool]:
    """-> (checkpoint, strict): --weights, else path.pretrain_model_G, loaded with path.strict_load."""
    path = args.weights if args.weights is not None else opts.pretrain_model_G
    if path is None:
        raise BinB200Error("path.pretrain_model_G: not set in the yml; give the weights with --weights")
    return path, opts.strict_load


def select_gpu(gpu_id: Optional[str], environ) -> Optional[str]:
    """demo.py:117: --gpu_id becomes CUDA_VISIBLE_DEVICES, outside torchrun; under torchrun (WORLD_SIZE > 1) it is
    ignored.  -> the message to print, if any.  Call before CUDA is initialised."""
    if gpu_id is None:
        return None
    if int(environ.get("WORLD_SIZE", "1")) > 1:
        return f"--gpu_id {gpu_id} is ignored under torchrun: rank r runs on GPU LOCAL_RANK"
    environ["CUDA_VISIBLE_DEVICES"] = str(gpu_id)
    return None


def main(argv=None) -> None:
    args = parse_args(argv)
    opts = load_options(args.opt)
    weights, strict = weights_of(args, opts)
    demo_py_steps(args.time_step)
    msg = select_gpu(args.gpu_id, os.environ)
    distributed = int(os.environ.get("WORLD_SIZE", "1")) > 1
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if msg is not None and int(os.environ.get("RANK", "0")) == 0:
        print(msg)
    torch.cuda.set_device(local)
    if distributed:
        torch.distributed.init_process_group("nccl", device_id=torch.device("cuda", local))
    try:
        net = rdn.bin_stage4_lstm()
        if args.arch is not None:
            net.model = rdn.RDN_residual_interp_5_input(lstm=True, GO=args.arch[0], D=args.arch[1])
        load_weights(net, weights, strict=strict)
        net = net.to(f"cuda:{local}").eval()
        bdist.broadcast_weights(net)
        rdn.set_precision(net, args.precision)
        rdn.set_self_ensemble(net, "flipx4" if args.flipx4 else None)
        run_demo(net, args.input_path, args.output_path, time_step=args.time_step,
                 decode_threads=args.decode_threads, model_path=weights)
    finally:
        if distributed:
            torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main()
