"""What the guarded optimizer step costs (DESIGN §4i): bin_adam_step against bin_grad_audit + bin_adam_step_guarded on the
network's 540 tensors, then the batch 8 x 256x256 training step of tools/bench_train.py with the guard off and on.
CUDA events; the two variants alternate so that both see the same clocks and neighbours.  Prints one JSON line with the
card's name and power limit, read in the same run.  There is no CPU path."""
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
if not torch.cuda.is_available():
    sys.exit("bench_guard: needs a CUDA device")
from bin_b200 import rdn  # noqa: E402
from bin_b200._lib import check, lib  # noqa: E402
from bin_b200.loss import pixel_loss  # noqa: E402
from bin_b200.optim import AUDIT_DTYPE, Adam  # noqa: E402
from oracle import bin_oracle as O  # noqa: E402

LAUNCHES, WARM, BLOCK = 200, 20, 20                     # kernel level: 200 timed launches per variant, in blocks of 20
B, H, W = (int(v) for v in sys.argv[1:4]) if len(sys.argv) > 3 else (8, 256, 256)
STEPS, ROUNDS = int(os.environ.get("BG_STEPS", 5)), 2


def timed(fn, n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                      capture_output=True, text=True).stdout.strip()
res = {"card": torch.cuda.get_device_name(0), "nvidia_smi_name_power_limit": card}

# ---- the optimizer's launches alone, on the real net's tensors
net = rdn.bin_stage4_lstm()
net.load_state_dict(O.synth_state_dict(0), strict=True)
net = net.cuda().train()
ps = list(net.parameters())
twins = [torch.nn.Parameter(p.detach().clone()) for p in ps]     # 260 steps on one gradient would wreck the net's own
for p in twins:
    p.grad = torch.randn_like(p) * 1e-3
opt = Adam(twins, lr=1e-4, betas=(0.9, 0.99))
opt.step()                                             # builds and uploads the table
tab = opt._tables[(0, 0)]
st = torch.cuda.current_stream().cuda_stream
rec = torch.zeros(AUDIT_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
scratch = torch.empty(lib().bin_grad_audit_scratch_bytes(tab.nchunks), dtype=torch.uint8, device="cuda")
adam_args = (tab.dev.data_ptr(), tab.prefix.data_ptr(), tab.n, tab.nchunks, 1e-4, 0.9, 0.99, 1e-8, 0.0, 0.1, 0.01, 1.0)


def plain():
    check(lib().bin_adam_step(*adam_args, st))


def audit():
    check(lib().bin_grad_audit(tab.dev.data_ptr(), tab.prefix.data_ptr(), tab.n, tab.nchunks, 1.0, 1.0, scratch.data_ptr(),
                               scratch.numel(), rec.data_ptr(), st))


def guarded():
    audit()
    check(lib().bin_adam_step_guarded(*adam_args, rec.data_ptr(), st))


for fn in (plain, guarded, audit):
    timed(fn, WARM)
ms = {"plain": 0.0, "guarded": 0.0, "audit": 0.0}
for _ in range(LAUNCHES // BLOCK):
    for name, fn in (("plain", plain), ("guarded", guarded), ("audit", audit)):
        ms[name] += timed(fn, BLOCK)
n = sum(p.numel() for p in ps)
res.update({"params": n, "tensors": len(ps), "launches_per_variant": LAUNCHES,
            "adam_step_us": round(1e3 * ms["plain"] / LAUNCHES, 2),
            "audit_plus_guarded_step_us": round(1e3 * ms["guarded"] / LAUNCHES, 2),
            "audit_alone_us": round(1e3 * ms["audit"] / LAUNCHES, 2),
            "audit_GBps_algorithmic": round(n * 4 / (ms["audit"] / LAUNCHES) / 1e6, 1)})      # 4 B read per gradient element

# ---- the whole training step, guard off and on, over the same parameters
fr = [f.cuda() for f in O.synth_frames(6, B, H, W, seed=1234, smooth=True)]
gt = [f.cuda() for f in O.synth_frames(14, B, H, W, seed=4321, smooth=True)]
opts = {"guard_off": Adam(ps, lr=1e-4, betas=(0.9, 0.99)),
        "guard_on": Adam(ps, lr=1e-4, betas=(0.9, 0.99), max_grad_norm=1e9, skip_nonfinite=True)}


def step_with(o):
    def step():
        o.zero_grad(set_to_none=True)
        loss, _ = pixel_loss(net(*fr), gt, "l1")
        loss.backward()
        o.step()
    return step


for o in opts.values():
    timed(step_with(o), 2)
rounds = {k: [] for k in opts}
for _ in range(ROUNDS):
    for k, o in opts.items():
        rounds[k].append(round(timed(step_with(o), STEPS) / STEPS, 2))
opts["guard_on"].resolve()
res.update({"train_step": f"batch {B} x {H}x{W}, forward + loss + backward + Adam, {STEPS} steps per round",
            "train_step_ms_guard_off": rounds["guard_off"], "train_step_ms_guard_on": rounds["guard_on"],
            "skipped_steps": opts["guard_on"].skipped_steps, "last_grad_norm": opts["guard_on"].last_grad_norm})
print(json.dumps(res))
