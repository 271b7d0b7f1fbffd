"""compute-sanitizer target: the fused RDB tail kernel and the x-stacked conv on small
tensors that still exercise several tiles per CTA (ntiles > #SMs), partial tiles in x and y, and a batch > 1.
usage: compute-sanitizer --tool {memcheck,racecheck,synccheck} python tools/sanitize_tail.py"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bin_b200 import ops  # noqa: E402

gen = torch.Generator(device="cuda").manual_seed(0)
rnd = lambda *sh: torch.randn(*sh, device="cuda", generator=gen)
for (B, H, W) in [(1, 6, 45), (2, 41, 290)]:            # 4 tiles / 2 x 11 x 10 = 220 tiles (> 148 CTAs: 2 tiles on 72 CTAs)
    x, g = rnd(B, 12, H, W, 8).half(), rnd(B, 16, H, W, 8).half()
    w3, wl = rnd(32, 192, 3, 3) / 1728 ** 0.5, rnd(96, 224, 1, 1) / 224 ** 0.5
    b3, bl = ops.pad_bias(rnd(32) * 0.1, 32), ops.pad_bias(rnd(96) * 0.1, 96)
    p3, pl = ops.pack_conv_weight(w3, 32, 192), ops.pack_conv_weight(wl, 96, 224)
    out = torch.zeros(B, 12, H, W, 8, device="cuda").half()
    g_ref, out_ref = g.clone(), out.clone()
    ops.rdb_tail_fwd(x, g, p3, b3, pl, bl, out)
    ops.conv_fwd(x, p3, b3, 3, 32, in0_planes=12, in1=g_ref, in1_planes=12, relu=True, out=g_ref, out_plane0=12)
    ops.conv_fwd(x, pl, bl, 1, 96, in0_planes=12, in1=g_ref, in1_planes=16, out=out_ref, res=x)
    torch.cuda.synchronize()
    print(f"B{B} {H}x{W}: fused == layerwise: {bool(torch.equal(out, out_ref))}", flush=True)
