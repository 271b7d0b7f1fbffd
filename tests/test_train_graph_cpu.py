"""The captured training step without a device: the --cuda_graph flag, its refusals (more than one rank, and
loss_scale_backoff with a capturable optimizer), BIN_B200_GRAPH=0, and the device-scalar block's layout against the
header."""
import os
import subprocess
import tempfile

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_graph_mode_switch(monkeypatch):
    from bin_b200 import BinB200Error
    from bin_b200.train import graph_mode
    monkeypatch.delenv("BIN_B200_GRAPH", raising=False)
    assert graph_mode(True, 1) and not graph_mode(False, 1) and not graph_mode(False, 4)
    monkeypatch.setenv("BIN_B200_GRAPH", "0")
    assert not graph_mode(True, 1)
    with pytest.raises(BinB200Error, match="one GPU"):
        graph_mode(True, 2)


def test_command_line_refuses_graph_with_ranks(monkeypatch, tmp_path):
    from bin_b200 import BinB200Error
    from bin_b200 import train as T
    monkeypatch.setenv("WORLD_SIZE", "2")
    with pytest.raises(BinB200Error, match="one GPU"):
        T.main(["-opt", str(tmp_path / "absent.yml"), "--cuda_graph"])   # refused before the options are read


def test_command_line_parses_the_flag(monkeypatch):
    from bin_b200 import train as T
    seen = {}

    class Stop(Exception):
        pass

    def fake(path):
        seen["path"] = path
        raise Stop
    monkeypatch.setattr(T, "load_options", fake)
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    with pytest.raises(Stop):
        T.main(["-opt", "x.yml", "--cuda_graph"])
    assert seen["path"] == "x.yml"


def test_capturable_refuses_loss_scale_backoff():
    from bin_b200.optim import Adam
    p = [torch.nn.Parameter(torch.zeros(3))]
    with pytest.raises(ValueError, match="capturable"):
        Adam(p, skip_nonfinite=True, loss_scale_backoff=True, capturable=True)
    opt = Adam(p, skip_nonfinite=True, capturable=True)
    assert opt.capturable and opt.resolve() is None and opt.skipped_steps == 0
    assert not Adam(p).capturable


def test_scalar_block_layout_matches_the_header():
    from bin_b200.optim import _LR, _STEP, SCALARS_DTYPE
    fields = list(SCALARS_DTYPE.names)
    src = ['#include <stddef.h>', '#include <stdio.h>', '#include "bin_b200.h"', 'int main(void) {',
           '  printf("size %zu\\n", sizeof(bin_adam_scalars_t));']
    src += [f'  printf("{f} %zu\\n", offsetof(bin_adam_scalars_t, {f}));' for f in fields]
    src += ['  return 0;', '}']
    with tempfile.TemporaryDirectory() as d:
        c, exe = os.path.join(d, "a.c"), os.path.join(d, "a.out")
        open(c, "w").write("\n".join(src))
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        got = dict(line.split() for line in subprocess.check_output([exe], text=True).splitlines())
    assert int(got["size"]) == SCALARS_DTYPE.itemsize == 48
    for f in fields:
        assert int(got[f]) == SCALARS_DTYPE.fields[f][1], f
    assert SCALARS_DTYPE.fields["lr"][1] == 4 * _LR and SCALARS_DTYPE.fields["step"][1] == 4 * _STEP


def test_adam_step_rejects_misaligned_scalars_before_any_launch():
    from bin_b200 import _lib
    L = _lib.lib()
    assert L.bin_adam_step(4096, 4096, 1, 1, 0.0, 0.9, 0.99, 1e-8, 0.0, 1.0, 1.0, 1.0, 4096 + 4, None) == 1
    assert "aligned" in L.bin_last_error().decode()
    assert L.bin_adam_step(4096, 4096, 0, 1, 0.0, 0.9, 0.99, 1e-8, 0.0, 1.0, 1.0, 1.0, 4096, None) == 1
