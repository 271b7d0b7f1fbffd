"""Generate tests/golden/ensemble.npz by EXECUTING THE REFERENCE'S OWN x4 flip self-ensemble (CPU; needs the reference
checkout with cv2 importable):

    python oracle/make_golden_ensemble.py /path/to/BIN

``utils/test_util.py:110-132 flipx4_forward`` runs unmodified on the reference's own ``models/archs/RDN.py`` net with
``bin_oracle.synth_state_dict(0)`` loaded strictly.  The helper passes ONE tensor to the model and keeps ``output[0]``
of a tuple, so the net is wrapped: it takes the six frames stacked as (6,B,3,H,W) and returns its 14 outputs stacked as
one (14,B,3,H,W) tensor.  ``torch.flip(inp, (-1,))`` etc. then flip every frame, and all 14 outputs are kept.  Two
cases: 32x48 B=1 and 18x26 B=2 (tile remainders at the half resolution 9x13, W not a multiple of 4).  The frames are
``bin_oracle.synth_frames(seed)``; the fixture stores their seed and a SHA-256 of their bytes instead of the frames, to
stay small.  Only the tensors the reference computes are stored; nothing of the reference is copied.
"""
import hashlib
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(os.path.dirname(HERE), "tests", "golden", "ensemble.npz")
CASES = {"a": (1, 32, 48, 4321), "b": (2, 18, 26, 4322)}        # B, H, W, frame seed


class Stacked(torch.nn.Module):
    """(6,B,3,H,W) -> (14,B,3,H,W): the window net behind the one-tensor interface flipx4_forward expects."""

    def __init__(self, net):
        super().__init__()
        self.net = net

    def forward(self, x):
        return torch.stack(self.net(*x.unbind(0)))


def main(ref_root):
    sys.path.insert(0, os.path.dirname(HERE))
    sys.path.insert(0, ref_root)
    import models.archs.RDN as R                   # the reference itself
    from utils.test_util import flipx4_forward     # the reference's own ensemble helper
    from oracle import bin_oracle as O
    torch.set_num_threads(os.cpu_count())
    net = R.bin_stage4_lstm().eval()
    res = net.load_state_dict(O.synth_state_dict(0), strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    model = Stacked(net).eval()
    rec = {}
    for tag, (B, H, W, seed) in CASES.items():
        fr = torch.stack(O.synth_frames(6, B, H, W, seed=seed, smooth=True))
        out = flipx4_forward(model, fr)
        assert out.shape == (14, B, 3, H, W)
        rec[f"{tag}_meta"] = np.array([B, H, W, seed])
        rec[f"{tag}_frames_sha256"] = np.array(hashlib.sha256(fr.numpy().tobytes()).hexdigest())
        rec[f"{tag}_out"] = out.numpy()
        print(tag, (B, H, W), "output range", float(out.min()), float(out.max()))
    np.savez_compressed(OUT, **rec)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main(sys.argv[1])
