"""Drop-in check against the reference's OWN model factory and checkpoint code.  tests/golden/reference_define_g.json
holds what the unmodified reference produced (oracle/make_golden_define_g.py): the class models.networks.define_G
builds for which_model_G 'bin_stage4' (networks.py:5-14), its state_dict key order, shapes and dtypes, and the keys
BaseModel.save_network writes (base_model.py:79-87).  Our factory must build the same schema, and a checkpoint in that
format with the 'InterpNet.' prefix that base_model.load_network strips (base_model.py:89-103) must strict-load."""
import hashlib
import json
import os

import torch


def _sha(lines):
    return hashlib.sha256("\n".join(lines).encode()).hexdigest()


def test_define_g_and_checkpoint_roundtrip(tmp_path, golden_dir):
    from oracle import bin_oracle as O
    import bin_b200.rdn as ours
    g = json.load(open(os.path.join(golden_dir, "reference_define_g.json")))
    netG = ours.bin_stage4_lstm()                                   # what define_G calls (networks.py:9-10)
    assert isinstance(netG, ours.RDN_residual_interp_5_input_ConvLSTM_L) and type(netG).__name__ == g["class"]
    sd = netG.state_dict()
    keys = list(sd.keys())
    assert len(keys) == g["n_keys"] and keys[:3] == g["first_keys"] and keys[-3:] == g["last_keys"]
    assert _sha(keys) == g["keys_sha256"]
    assert _sha([f"{k}:{tuple(v.shape)}:{v.dtype}" for k, v in sd.items()]) == g["shapes_sha256"]
    # checkpoint round trip: a file in the reference's format, loaded the way load_network does
    ckpt = tmp_path / "ck_G.pth"
    torch.save({("InterpNet." + k): v for k, v in O.synth_state_dict(2).items()}, ckpt)
    clean = {(k[len("InterpNet."):] if k.startswith("InterpNet.") else k): v for k, v in torch.load(ckpt).items()}
    netG.load_state_dict(clean, strict=True)
    assert torch.equal(netG.model.model2_3.GFF[0].weight, O.synth_state_dict(2)["model.model2_1.GFF.0.weight"])
    # save_network writes state_dict() as is: the same keys the reference's own network writes
    torch.save(netG.state_dict(), tmp_path / "7_G.pth")
    assert _sha(list(torch.load(tmp_path / "7_G.pth").keys())) == g["saved_keys_sha256"]
