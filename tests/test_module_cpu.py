"""CPU-side checks of the drop-in boundary (SURVEY 8b): schema, strict load, loud failure
without CUDA, and that the C-ABI library exports every symbol the header declares."""
import os
import re

import pytest
import torch

from oracle import bin_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def net():
    from bin_b200 import rdn
    torch.manual_seed(0)
    return rdn.bin_stage4_lstm()


def test_state_dict_schema_matches_reference(net):
    sd_ref = O.synth_state_dict(0)            # key order + shapes were asserted against the reference in make_golden.py
    sd = net.state_dict()
    assert list(sd.keys()) == list(sd_ref.keys())
    for k in sd:
        assert tuple(sd[k].shape) == tuple(sd_ref[k].shape), k
    assert len(sd) == 1332
    uniq = list(net.parameters())
    assert len(uniq) == 540 and sum(p.numel() for p in uniq) == 11_441_668


def test_strict_load_and_aliasing(net):
    sd_ref = O.synth_state_dict(3)
    res = net.load_state_dict(sd_ref, strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    m = net.model
    assert m.model1_2 is m.model1_1 and m.model1_4 is m.model1_1 and m.model2_3 is m.model2_1 and m.model3_2 is m.model3_1
    assert torch.equal(m.model1_3.SFENet1.weight, sd_ref["model.model1_1.SFENet1.weight"])


def test_prefix_stripping_like_base_model(net):
    """base_model.load_network strips 'module.' / 'InterpNet.' prefixes then loads strictly (base_model.py:89-103)."""
    sd_ref = O.synth_state_dict(1)
    wrapped = {"module." + k: v for k, v in sd_ref.items()}
    clean = {k[7:] if k.startswith("module.") else k: v for k, v in wrapped.items()}
    net.load_state_dict(clean, strict=True)


def test_cpu_forward_fails_loudly(net):
    from bin_b200 import BinB200Error
    fr = O.synth_frames(6, 1, 16, 16)
    with torch.no_grad(), pytest.raises(BinB200Error):
        net(*fr)


def test_grad_path_on_cpu_fails_loudly(net):
    """Training goes through the same CUDA library: a grad-enabled CPU call must raise, not fall back."""
    from bin_b200 import BinB200Error
    fr = O.synth_frames(6, 1, 16, 16)
    with pytest.raises(BinB200Error):
        net(*fr)


def test_library_exports_every_declared_symbol():
    import ctypes
    from bin_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "bin_b200.h")).read()
    declared = set(re.findall(r"\b(bin_[a-z0-9_]+)\s*\(", hdr))
    declared -= {"bin_b200"}
    L = ctypes.CDLL(_lib.LIB_PATH)
    for name in sorted(declared):
        assert hasattr(L, name), f"{name} declared in include/bin_b200.h but not exported"
    assert declared == set(_lib.exported_symbols()), declared ^ set(_lib.exported_symbols())
    assert _lib.lib().bin_abi_version() == _lib.ABI_VERSION == int(re.search(r"#define BIN_ABI_VERSION (\d+)", hdr).group(1))
    # measurement tooling (microbenchmarks, debug timelines) is never part of the product library or its header
    assert not any(n.startswith(("bin_tools_", "bin_microbench", "bin_debug")) for n in declared)
    assert not hasattr(L, "bin_tools_microbench_mma") and not hasattr(L, "bin_microbench_mma")


def test_workspace_queries_are_pure():
    from bin_b200 import _lib
    L = _lib.lib()
    assert L.bin_backbone_packed_bytes(2) > 5_000_000 and L.bin_backbone_packed_bytes(4) == 0
    a = L.bin_backbone_workspace_bytes(2, 1, 64, 64)
    assert 0 < a < L.bin_backbone_workspace_bytes(2, 1, 128, 128)


def test_convlstm_cell_table_is_checked_before_any_launch():
    """bin_convlstm_fwd refuses a bad cell table with BIN_ERR_ARG before it launches (the pointers are fake and never
    dereferenced)."""
    from bin_b200 import _lib
    L = _lib.lib()
    p = 1 << 20

    def call(cells, n=None):
        tab = (_lib.LstmCell * len(cells))(*[_lib.LstmCell(*c) for c in cells])
        rc = L.bin_convlstm_fwd(tab if cells else None, len(cells) if n is None else n, 1, 8, 8, None)
        return rc, L.bin_last_error().decode()

    plain, stateful = (p, None, None, p, p, p, None), (p, p, p, p, p, p, p)
    assert call([]) == (1, "convlstm: null cell table")
    assert call([plain], 0) == (1, "convlstm: 1..3 cells per launch")
    assert call([plain] * 4) == (1, "convlstm: 1..3 cells per launch")
    assert call([plain, (p, None, None, p, p, None, None)]) == (1, "convlstm: null argument")
    assert call([(p, p, None, p, p, p, None)]) == (1, "convlstm: give both c_prev and h_prev or neither")
    assert call([stateful, plain]) == (1, "convlstm: cells of one launch must all have or all lack a state")


def test_wgrad_rejects_bad_segments_before_any_launch():
    """bin_conv_wgrad checks its segments on the host: TMA zero-fills a box that runs past its tensor, so a plane range
    or geometry error would otherwise come back as quietly wrong gradients.  Every call here is invalid and must fail
    with BIN_ERR_ARG before a tensor map is built (the tensors are null: nothing reaches a device)."""
    import ctypes as C
    from bin_b200 import _lib
    L = _lib.lib()
    act = lambda planes, B=2, H=9, W=20: _lib.Act(None, B, planes, H, W)
    none = _lib.Act(None, 0, 0, 0, 0)
    ws = (C.c_float * 1)()
    cases = [  # (x0, x0_plane0, x0_planes, x1, x1_plane0, x1_planes, dy, dy_plane0, cout, cin, ks), error text
        ((act(12), 0, 0, none, 0, 0, act(4), 0, 32, 96, 3), "plane counts"),
        ((act(12), 0, 6, none, 0, 0, act(4), 0, 32, 48, 3), "plane counts"),
        ((act(144), 12, 12, act(192), 16, 6, act(16), 4, 32, 144, 3), "plane counts"),
        ((act(12), 0, 12, act(16), 0, -4, act(16), 0, 32, 96, 3), "plane counts"),
        ((act(144), 136, 12, none, 0, 0, act(16), 0, 32, 96, 3), "plane range"),
        ((act(144), -4, 12, none, 0, 0, act(16), 0, 32, 96, 3), "plane range"),
        ((act(144), 12, 12, act(192), 180, 16, act(144), 12, 96, 224, 1), "plane range"),
        ((act(12), 0, 12, act(16, H=8), 0, 16, act(12), 0, 96, 224, 1), "geometry"),
        ((act(12), 0, 12, act(16, B=3), 0, 16, act(12), 0, 96, 224, 1), "geometry"),
        ((act(12), 0, 12, none, 0, 0, act(12, W=21), 0, 96, 96, 3), "geometry"),
        ((act(12), 0, 12, none, 0, 0, act(12, B=1), 0, 96, 96, 3), "geometry"),
        ((act(144), 12, 12, act(192), 16, 4, act(16), 4, 32, 160, 3), "Cin exceeds"),
        ((act(4), 0, 4, none, 0, 0, act(12), 0, 96, 36, 5), "Cin exceeds"),
        ((act(12), 0, 12, none, 0, 0, act(16), 14, 32, 96, 3), "dY plane range"),
        ((act(12), 0, 12, none, 0, 0, act(16), -1, 32, 96, 3), "dY plane range"),
    ]
    for args, text in cases:
        rc = L.bin_conv_wgrad(*args, None, None, C.addressof(ws), None)
        err = L.bin_last_error().decode()
        assert rc == 1 and text in err and err.startswith("wgrad:"), (args[1:3], args[4:6], args[7:], rc, err)


def test_conv_fwd_rejects_bad_arguments_before_any_launch():
    """bin_conv_fwd checks every argument on the host before it builds a tensor map: a plane range past a tensor would
    otherwise be zero-filled by TMA (reads) or written past its end (stores), and an option the selected kernel does not
    apply would be dropped without a word.  Every call here is invalid and must fail with BIN_ERR_ARG.  The geometry
    cases pass null pointers only; the pointer cases point the non-null arguments at a small host buffer, and each of
    them still has a null pointer, so nothing reaches a device."""
    import ctypes as C
    from bin_b200 import _lib
    L = _lib.lib()
    buf = (C.c_double * 8)()                        # host memory, never dereferenced
    hp = (C.addressof(buf) + 15) & ~15
    act = lambda planes, B=2, H=9, W=20, ptr=None: _lib.Act(ptr, B, planes, H, W)
    res = lambda planes, B=2: act(planes, B=B, ptr=hp)   # a residual is present iff its pointer is set

    def args(**kw):
        a = _lib.ConvArgs()
        a.in0, a.in0_planes, a.ksize, a.cout_pad, a.epilogue = act(12), 12, 1, 96, _lib.EPI_P8
        a.out = act(12)
        for k, v in kw.items():
            setattr(a, k, v)
        return a
    x3 = dict(x3=1)
    cases = [  # (fields, error text)
        # plane counts, negative offsets, x3 alignment
        (dict(in0_planes=0), "plane counts"),
        (dict(in0_planes=6), "plane counts"),
        (dict(in1=act(16), in1_planes=-4), "plane counts"),
        (dict(in0=act(24), in0_plane0=-4), "negative plane offset"),
        (dict(in1=act(16), in1_plane0=-4, in1_planes=4), "negative plane offset"),
        (dict(out=act(24), out_plane0=-12), "negative plane offset"),
        (dict(res=res(24), res_plane0=-12), "negative plane offset"),
        (dict(store_planes=-1), "negative plane offset"),
        (dict(epilogue=_lib.EPI_PIXSHUF, ksize=3, cout_pad=256, out=act(8, H=18, W=40), out_plane0=-4), "negative plane offset"),
        (dict(in0=act(24), in0_plane0=2, **x3), "multiples of 4"),
        # input ranges and geometry
        (dict(in0=act(12), in0_plane0=4), "input plane range"),
        (dict(in0=act(20), in0_planes=12, **x3), "input plane range"),
        (dict(in1=act(16), in1_plane0=8, in1_planes=12), "input plane range"),
        (dict(in1=act(16, H=8), in1_planes=16), "in1 geometry"),
        (dict(in1=act(16, B=3), in1_planes=4), "in1 geometry"),
        # sub-ranges
        (dict(b_begin=2), "sub-range"),
        (dict(b_begin=1, b_count=2), "sub-range"),
        (dict(y_begin=-1), "sub-range"),
        (dict(y_begin=5, y_count=5), "sub-range"),
        (dict(b_count=-1), "sub-range"),
        # output / residual ranges; x3: the last logical plane's lo half must lie inside the tensor
        (dict(out=act(11)), "output tensor geometry"),
        (dict(out=act(24), out_plane0=13), "output tensor geometry"),
        (dict(out=act(12, W=21)), "output tensor geometry"),
        (dict(store_planes=13), "output tensor geometry"),
        (dict(in0=act(24), out=act(20), **x3), "output tensor geometry"),                       # 4 planes short
        (dict(in0=act(24), out=act(28), out_plane0=12, store_planes=1, **x3), "output tensor geometry"),   # needs 29
        (dict(in0=act(24), out=act(24), res=res(20), **x3), "residual tensor geometry"),
        (dict(in0=act(24), out=act(24), res=res(284), res_plane0=132, **x3), "residual tensor geometry"),
        (dict(res=res(24), res_plane0=13), "residual tensor geometry"),
        (dict(res=res(12, B=1)), "residual tensor geometry"),
        (dict(epilogue=_lib.EPI_PIXSHUF, ksize=3, cout_pad=256, out=act(7, H=18, W=40)), "pixel-shuffle output"),
        (dict(epilogue=_lib.EPI_PIXSHUF, ksize=3, cout_pad=256, out=act(8, H=9, W=40)), "pixel-shuffle output"),
        (dict(epilogue=_lib.EPI_PIXSHUF, ksize=3, cout_pad=256, in0=act(24), out=act(12, H=18, W=40), **x3),
         "pixel-shuffle output"),
        # options the selected kernel would drop
        (dict(ksize=3, cout_pad=32, out=act(4), res=res(4), relu=1), "takes no residual"),
        (dict(ksize=3, cout_pad=32, in0=act(24), out=act(8), res=res(8), **x3), "takes no residual"),
        (dict(epilogue=_lib.EPI_PIXSHUF, ksize=3, cout_pad=256, out=act(8, H=18, W=40), relu=1), "no ReLU and no residual"),
        (dict(epilogue=_lib.EPI_PIXSHUF, ksize=3, cout_pad=256, out=act(8, H=18, W=40), res=res(12)), "no ReLU and no residual"),
        (dict(epilogue=_lib.EPI_FINAL, ksize=3, cout_pad=16, relu=1), "no ReLU and no residual"),
        (dict(epilogue=_lib.EPI_FINAL, ksize=3, cout_pad=16, res=res(12)), "no ReLU and no residual"),
        # the final epilogue's frame table
        (dict(epilogue=_lib.EPI_FINAL, ksize=3, cout_pad=16), "frame table"),
        # null pointers, once every shape is right
        (dict(), "null input tensor"),
        (dict(in0=act(12, ptr=hp), in1=act(16), in1_planes=16), "null input tensor"),
        (dict(in0=act(12, ptr=hp + 8)), "16-byte aligned"),
        (dict(in0=act(12, ptr=hp)), "null weights or bias"),
        (dict(in0=act(12, ptr=hp), w_packed=hp), "null weights or bias"),
        (dict(in0=act(12, ptr=hp), bias=hp), "null weights or bias"),
        (dict(in0=act(12, ptr=hp), w_packed=hp, bias=hp), "null output tensor"),
        (dict(epilogue=_lib.EPI_PIXSHUF, ksize=3, cout_pad=256, in0=act(12, ptr=hp), w_packed=hp, bias=hp,
              out=act(8, H=18, W=40)), "null output tensor"),
    ]
    for fields, text in cases:
        a = args(**fields)
        rc = L.bin_conv_fwd(C.byref(a), None)
        err = L.bin_last_error().decode()
        assert rc == 1 and text in err and err.startswith("conv:"), (fields, rc, err)
    # FINAL: a frame table that matches the batch but holds a null frame or output pointer
    for null_out in (False, True):
        a = args(epilogue=_lib.EPI_FINAL, ksize=3, cout_pad=16, in0=act(12, ptr=hp), w_packed=hp, bias=hp)
        a.fr.ncalls, a.fr.nframes, a.fr.Bc = 2, 3, 1
        for k in range(2):
            a.fr.out[k] = None if (null_out and k == 1) else hp
            for f in range(3):
                a.fr.frame[k][f] = None if (not null_out and (k, f) == (1, 2)) else hp
        rc = L.bin_conv_fwd(C.byref(a), None)
        err = L.bin_last_error().decode()
        assert rc == 1 and "null frame or output" in err, (null_out, rc, err)


def test_rdb_tail_rejects_bad_planes_before_any_launch():
    """bin_rdb_tail_fwd: negative plane offsets and ranges past a tensor fail with BIN_ERR_ARG (null pointers only)."""
    import ctypes as C
    from bin_b200 import _lib
    L = _lib.lib()
    act = lambda planes, B=2, H=9, W=20: _lib.Act(None, B, planes, H, W)
    cases = [  # (x, x_plane0, g, g_plane0, out, out_plane0, sub), error text
        ((act(144), -12, act(192), 0, act(144), 0, (0, 0, 0, 0)), "plane range"),
        ((act(144), 0, act(192), -16, act(144), 12, (0, 0, 0, 0)), "plane range"),
        ((act(144), 0, act(192), 0, act(144), -12, (0, 0, 0, 0)), "plane range"),
        ((act(144), 133, act(192), 0, act(144), 0, (0, 0, 0, 0)), "plane range"),
        ((act(144), 0, act(192), 181, act(144), 12, (0, 0, 0, 0)), "plane range"),
        ((act(144), 0, act(192), 0, act(144, H=8), 12, (0, 0, 0, 0)), "geometry"),
        ((act(144), 0, act(192), 0, act(144), 12, (0, 0, 9, 0)), "sub-range"),
        ((act(144), 0, act(192), 0, act(144), 12, (0, 0, 0, 0)), "null argument"),
    ]
    for (x, xp, g, gp, out, op, sub), text in cases:
        rc = L.bin_rdb_tail_fwd(C.byref(x), xp, C.byref(g), gp, None, None, None, None, C.byref(out), op, *sub, None)
        err = L.bin_last_error().decode()
        assert rc == 1 and text in err and err.startswith("rdb_tail"), (xp, gp, op, sub, rc, err)


def test_precision_pack_entry_points_check_prec():
    import ctypes as C
    from bin_b200 import _lib
    L = _lib.lib()
    fr = _lib.Frames()
    assert L.bin_pack_frames_p(C.byref(fr), 4, 4, _lib.Act(None, 1, 8, 2, 2), 2, None) == 1
    assert "precision" in L.bin_last_error().decode()
    assert L.bin_pack_conv_weight_p(None, 96, 96, 3, 96, 96, 0, -1, None, None) == 1
    assert "precision" in L.bin_last_error().decode()


def test_training_side_modules_refuse_cpu_tensors():
    """bin_b200.optim / bin_b200.dataprep have no CPU path: they must say so instead of computing something."""
    import torch
    from bin_b200 import BinB200Error
    from bin_b200.dataprep import blur_average, window_count
    from bin_b200.optim import Adam
    p = torch.nn.Parameter(torch.ones(4))
    p.grad = torch.ones(4)
    opt = Adam([p], lr=1e-3, betas=(0.9, 0.99), weight_decay=1e-4)
    assert opt.param_groups[0]["betas"] == (0.9, 0.99) and opt.param_groups[0]["weight_decay"] == 1e-4
    with pytest.raises(BinB200Error):
        opt.step()
    assert torch.all(p == 1)
    with pytest.raises(ValueError):
        Adam([p], lr=-1.0)
    with pytest.raises(BinB200Error):
        blur_average(torch.zeros((40, 4, 4, 3), dtype=torch.uint8))
    # create_dataset_blur_N_frames_average.py:104  window_total_num = floor(n_length / 8) - 2
    assert [window_count(n) for n in (24, 40, 47, 48, 240)] == [1, 3, 3, 4, 28]


def test_ctypes_structs_match_the_header_layout(tmp_path):
    """sizeof / offsetof of every ABI struct as gcc sees include/bin_b200.h == the ctypes mirror in bin_b200/_lib.py
    (and the 5 x int64 rows bin_b200.optim uploads == bin_adam_tensor_t)."""
    import ctypes as C
    import subprocess
    from bin_b200 import _lib
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    probes = {"bin_act_t": (_lib.Act, ["ptr", "B", "planes", "H", "W"]),
              "bin_frames_t": (_lib.Frames, ["frame", "out", "ncalls", "nframes", "Bc"]),
              "bin_conv_args_t": (_lib.ConvArgs, [f[0] for f in _lib.ConvArgs._fields_]),
              "bin_lstm_cell_t": (_lib.LstmCell, ["x", "c_prev", "h_prev", "w", "b", "h_out", "c_out"])}
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "bin_b200.h"', 'int main(void) {']
    for cname, (_, fields) in probes.items():
        lines.append(f'  printf("{cname} %zu\\n", sizeof({cname}));')
        for f in fields:
            lines.append(f'  printf("{cname}.{f} %zu\\n", offsetof({cname}, {f}));')
    lines += ['  printf("bin_adam_tensor_t %zu\\n", sizeof(bin_adam_tensor_t));',
              '  printf("bin_adam_tensor_t.n %zu\\n", offsetof(bin_adam_tensor_t, n));', '  return 0;', '}']
    src = tmp_path / "probe.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "probe"
    subprocess.run(["gcc", "-I", os.path.join(root, "include"), str(src), "-o", str(exe)], check=True)
    got = dict(l.split() for l in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines())
    for cname, (ct, fields) in probes.items():
        assert int(got[cname]) == C.sizeof(ct), cname
        for f in fields:
            assert int(got[f"{cname}.{f}"]) == getattr(ct, f).offset, f"{cname}.{f}"
    assert int(got["bin_adam_tensor_t"]) == 5 * 8 and int(got["bin_adam_tensor_t.n"]) == 4 * 8


def test_weight_walk_matches_parameters_and_survives_replication(net):
    """nn.DataParallel replicas (bin_model.py:42) have EMPTY _parameters and carry their weights as plain attributes
    (torch/nn/parallel/replicate.py): the tensors handed to the C ABI must therefore be read from the conv modules, in
    the registration order bin_backbone_pack expects."""
    import torch
    for bb in (net.model.model1_1, net.model.model2_1, net.model.model3_1, net.model.model4_1):
        walked, regs = bb._conv_params(), list(bb.parameters())
        assert len(walked) == 132 and all(a is b for a, b in zip(walked, regs))
    allt = net._all_tensors()
    assert len(allt) == 540 and {id(t) for t in allt} == {id(p) for p in net.parameters()}
    # what replicate() does to one module tree, on CPU: copy every module, drop _parameters, set plain tensor attributes
    mods = list(net.modules())
    copies = {id(m): m._replicate_for_data_parallel() for m in mods}
    for m in mods:
        r = copies[id(m)]
        for key, child in m._modules.items():
            setattr(r, key, copies[id(child)])
        for key, p in m._parameters.items():
            setattr(r, key, p.detach() * 2.0)
    rep = copies[id(net)]
    assert len(list(rep.parameters())) == 0                       # the reason self.parameters() cannot be used
    rw = rep._all_tensors()
    assert len(rw) == 540 and all(torch.equal(a, b * 2.0) for a, b in zip(rw, allt))
    assert rep.model.model1_3 is rep.model.model1_1               # aliases stay aliases inside a replica


def test_bench_reference_arm_line_on_cpu():
    """`bench.py --impl reference` (the driver's reference arm) on a tiny window: one JSON line with the contract's keys,
    kind "reference" where the unmodified reference is mounted and "port" otherwise; a non-zero rank prints nothing."""
    import json
    import subprocess
    import sys
    cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--height", "48", "--width", "64",
           "--steps", "3", "--warmup", "1", "--gpus", "2"]
    env = dict(os.environ, RANK="0", WORLD_SIZE="2", LOCAL_RANK="0")
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [l for l in r.stdout.strip().split("\n") if l.startswith("{")]
    assert len(lines) == 1
    j = json.loads(lines[0])
    assert j["impl"] == "reference" and j["metric"] == "720p frame-windows/sec" and j["unit"] == "windows/s"
    assert j["higher_is_better"] is True and j["value"] > 0 and j["n_gpus"] == 2
    assert j["steps"] == 2 and j["requested_steps"] == 3            # bounded sample: at most two timed windows
    cb = j["cpu_baseline"]
    assert cb["kind"] in ("reference", "port") and cb["cores"] >= 1 and cb["value"] == j["value"] and cb["sample"]
    assert j["e2e"] == {"value": j["value"], "unit": "windows/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    r1 = subprocess.run(cmd, env=dict(env, RANK="1", LOCAL_RANK="1"), capture_output=True, text=True, timeout=600)
    assert r1.returncode == 0 and r1.stdout.strip() == ""


def test_bench_clock_sampler_uses_only_samples_of_the_timed_region():
    """bench.py's ClockSampler: median / min SM clock and throttle reasons come from the samples that arrived between
    mark_begin and mark_end (the sampler itself starts before the warm-up); without nvidia-smi it says so."""
    import importlib.util
    spec = importlib.util.spec_from_file_location("bench_mod", os.path.join(ROOT, "bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)

    class FakeProc:
        def terminate(self):
            pass
    s = bench.ClockSampler(0)
    s.proc = FakeProc()
    row = lambda mhz, cap: ["0", str(mhz), "1965", "700.0", "Not Active", "Not Active", "Not Active", cap]
    s.rows = [(10.0, row(1965, "Not Active")), (20.5, row(1500, "Active")), (21.0, row(1470, "Active")), (21.5, row(1530, "Active")),
              (40.0, row(600, "Not Active"))]
    s.t0, s.t1 = 20.0, 22.0
    r = s.stop()
    assert r["sm_mhz"] == 1500 and r["sm_min_mhz"] == 1470 and r["sm_max_mhz"] == 1965 and r["samples"] == 3
    assert r["reasons"] == ["sw_power_cap"]
    s2 = bench.ClockSampler(0)                        # nvidia-smi absent (this container)
    assert s2.stop()["reasons"] == ["nvidia-smi unavailable"]
    p = bench.peaks()
    assert p["bf16_tflops"] > 0 and p["hbm_gbs"] > 0 and p["source"] in ("measured", "fallback")
