"""Time one optimizer step over the network's 540 tensors: bin_b200.optim.Adam vs torch.optim.Adam (fused / foreach),
and the blur-synthesis kernel on a 640x352 clip.  CUDA events, 20 iterations after 3 warm-ups."""
import json
import sys

import torch

sys.path.insert(0, ".")
import bin_b200.rdn as RDN                      # noqa: E402
from bin_b200.dataprep import blur_average     # noqa: E402
from bin_b200.optim import Adam                # noqa: E402


def timed(fn, iters=20, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


net = RDN.bin_stage4_lstm().cuda()
ps = list(net.parameters())
for p in ps:
    p.grad = torch.randn_like(p) * 1e-3
n = sum(p.numel() for p in ps)
res = {"params": n, "tensors": len(ps)}
ours = Adam(ps, lr=1e-4, betas=(0.9, 0.99))
res["ours_ms"] = timed(ours.step)
tab = ours._tables[(0, 0)]
from bin_b200._lib import check, lib           # noqa: E402
st = torch.cuda.current_stream().cuda_stream
res["ours_kernel_ms"] = timed(lambda: check(lib().bin_adam_step(tab.dev.data_ptr(), tab.prefix.data_ptr(), tab.n, tab.nchunks,
                                                                1e-4, 0.9, 0.99, 1e-8, 0.0, 0.1, 0.01, 1.0, None, st)),
                                      iters=50)
res["torch_fused_ms"] = timed(torch.optim.Adam(ps, lr=1e-4, betas=(0.9, 0.99), fused=True).step)
res["torch_foreach_ms"] = timed(torch.optim.Adam(ps, lr=1e-4, betas=(0.9, 0.99), foreach=True).step)
res["ours_GBps_algorithmic"] = n * 28 / res["ours_kernel_ms"] / 1e6          # 16 B read + 12 B written per parameter

frames = torch.randint(0, 256, (240, 352, 640, 3), dtype=torch.uint8, device="cuda")
ms = timed(lambda: blur_average(frames, window_size=11))
nwin = 240 // 8 - 2
res["blur_ms"] = ms
res["blur_GBps_algorithmic"] = (frames.numel() + nwin * frames[0].numel()) / ms / 1e6    # each frame once + outputs
res["blur_GBps_l2_side"] = (11 + 1) * nwin * frames[0].numel() / ms / 1e6
print(json.dumps(res))
