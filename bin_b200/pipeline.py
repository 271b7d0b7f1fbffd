"""Host<->device pipelining of consecutive windows (the caller-side loop of test.py:249-402).

test.py uploads six frames, runs the net and downloads three images per window, serially on one
stream.  Windows are independent, so the upload of window k+1 and the download of window k-1 can
overlap the forward of window k: three CUDA streams + events, two rotating input slots.
"""
from __future__ import annotations

from collections import deque
from typing import List, Sequence

import torch


class WindowPipeline:
    """Copies back the window outputs `out_indices`; call rdn.set_outputs(net, out_indices) first so that the net
    computes only those."""

    def __init__(self, net: torch.nn.Module, device, out_indices: Sequence[int] = (13, 8, 12), slots: int = 2):
        self.net, self.dev, self.out_idx = net, torch.device(device), tuple(out_indices)
        self.s_in, self.s_out = torch.cuda.Stream(self.dev), torch.cuda.Stream(self.dev)
        self.slots = [None] * slots          # device input buffers, reused round-robin
        self.free_evt = [None] * slots       # compute finished reading slot i
        self.k = 0
        self.pending = deque()

    def submit(self, frames_host: Sequence[torch.Tensor], outs_host: Sequence[torch.Tensor]):
        """frames_host: 6 pinned (B,3,H,W) fp32 tensors; outs_host: pinned destinations for out_indices."""
        i = self.k % len(self.slots)
        self.k += 1
        main = torch.cuda.current_stream(self.dev)
        with torch.cuda.stream(self.s_in):
            if self.free_evt[i] is not None:
                self.s_in.wait_event(self.free_evt[i])
            if self.slots[i] is None or self.slots[i][0].shape != frames_host[0].shape:
                self.slots[i] = [torch.empty(f.shape, dtype=f.dtype, device=self.dev) for f in frames_host]
            for d, f in zip(self.slots[i], frames_host):
                d.copy_(f, non_blocking=True)
            up = torch.cuda.Event()
            up.record(self.s_in)
        main.wait_event(up)
        with torch.no_grad():
            outs = self.net(*self.slots[i])
        done = torch.cuda.Event()
        done.record(main)
        self.free_evt[i] = done
        with torch.cuda.stream(self.s_out):
            self.s_out.wait_event(done)
            for dst, k in zip(outs_host, self.out_idx):
                dst.copy_(outs[k], non_blocking=True)
                outs[k].record_stream(self.s_out)
            fin = torch.cuda.Event()
            fin.record(self.s_out)
        self.pending.append(fin)
        return fin

    def drain(self):
        while self.pending:
            self.pending.popleft().synchronize()
