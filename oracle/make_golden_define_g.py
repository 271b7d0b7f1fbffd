"""Writes tests/golden/reference_define_g.json from the unmodified reference (CPU; needs the reference checkout):

    python oracle/make_golden_define_g.py /path/to/BIN

the class models.networks.define_G builds for which_model_G 'bin_stage4', hashes of its state_dict key order and of
(key, shape, dtype), and a hash of the keys BaseModel.save_network writes.  Only these facts are stored."""
import hashlib
import json
import os
import sys
import tempfile

import torch

HERE = os.path.dirname(os.path.abspath(__file__))


def _sha(lines):
    return hashlib.sha256("\n".join(lines).encode()).hexdigest()


def main(ref_root):
    sys.path.insert(0, ref_root)
    import models.networks as networks
    from models.base_model import BaseModel
    netG = networks.define_G({"network_G": {"which_model_G": "bin_stage4", "nframes": 6, "version": 2}})
    sd = netG.state_dict()
    d = tempfile.mkdtemp()
    bm = BaseModel.__new__(BaseModel)
    bm.device = torch.device("cpu")
    bm.opt = {"path": {"models": d}}
    BaseModel.save_network(bm, netG, "G", 7)
    back = torch.load(os.path.join(d, "7_G.pth"))
    g = {"source": "reference models.networks.define_G({'network_G': {'which_model_G': 'bin_stage4'}}) and BaseModel.save_network, CPU",
         "class": type(netG).__name__, "n_keys": len(sd),
         "keys_sha256": _sha(list(sd.keys())),
         "shapes_sha256": _sha([f"{k}:{tuple(v.shape)}:{v.dtype}" for k, v in sd.items()]),
         "saved_keys_sha256": _sha(list(back.keys())),
         "first_keys": list(sd.keys())[:3], "last_keys": list(sd.keys())[-3:]}
    with open(os.path.join(HERE, "..", "tests", "golden", "reference_define_g.json"), "w") as fh:
        json.dump(g, fh, indent=1)


if __name__ == "__main__":
    main(sys.argv[1])
