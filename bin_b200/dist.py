"""Multi-GPU plumbing for the BIN hot path: one process per GPU, windows are the parallel unit (shard_windows deals them
round-robin; shard_test_set gives each rank a contiguous run, so streaming keeps its stage-1 reuse).

SURVEY.md 8e: every window's forward is a pure function of its 6 frames and the weights (state is
re-zeroed per call, RDN.py:423-434), so inference shards over windows with NO collective in the
loop; the only communication is one broadcast of the parameters from rank 0 at start-up (NCCL over
NVLink on GPUs, gloo in the CPU tests)."""
from __future__ import annotations

from typing import List, Mapping, Tuple

import torch
import torch.distributed as dist


def shard_windows(n_windows: int, rank: int, world: int) -> List[int]:
    """Window w -> rank w mod world (round-robin keeps consecutive frames spread evenly)."""
    return list(range(rank, n_windows, world))


def shard_test_set(lengths: Mapping[str, int], world: int) -> List[List[Tuple[str, range]]]:
    """Split a test set's windows into `world` contiguous pieces, one per rank, so each rank streams consecutive windows
    and keeps stage-1 reuse (streaming.stream_video).  lengths: folder name -> its number of blurry frames.  The windows
    are laid out in test.py's order (sorted folders, then windows 0 .. N-2 of each, test.py:158, 249-255) and cut into
    `world` runs whose window counts differ by at most 1; a run may span folders.  -> per rank, its (folder, range of
    window indices) pieces in that order.  A cut inside a folder costs at most 4 stage-1 calls and 5 frame decodes more
    than streaming the folder whole: the first window of a range reads up to five frames the range before also read."""
    if world < 1:
        raise ValueError(f"world must be >= 1, got {world}")
    folders = [(f, max(int(lengths[f]) - 1, 0)) for f in sorted(lengths)]
    total = sum(nw for _, nw in folders)
    cuts = [r * total // world for r in range(world + 1)]
    out: List[List[Tuple[str, range]]] = []
    for r in range(world):
        lo, hi, pieces, base = cuts[r], cuts[r + 1], [], 0
        for f, nw in folders:
            a, b = max(lo - base, 0), min(hi - base, nw)
            if a < b:
                pieces.append((f, range(a, b)))
            base += nw
        out.append(pieces)
    return out


def broadcast_weights(module: torch.nn.Module, src: int = 0) -> int:
    """One flat broadcast of the 540 unique tensors (11.44 M fp32 = 45.8 MB).  Returns bytes sent."""
    params = [p for p in module.parameters()]
    if not dist.is_available() or not dist.is_initialized() or dist.get_world_size() == 1:
        return 0
    flat = torch.cat([p.detach().reshape(-1) for p in params])
    dist.broadcast(flat, src=src)
    off = 0
    with torch.no_grad():
        for p in params:
            n = p.numel()
            p.copy_(flat[off:off + n].view_as(p))      # in-place: bumps ._version -> packed blobs refresh
            off += n
    return flat.numel() * flat.element_size()


def max_over_ranks(value: float, device) -> float:
    if not dist.is_available() or not dist.is_initialized() or dist.get_world_size() == 1:
        return value
    t = torch.tensor([value], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())
