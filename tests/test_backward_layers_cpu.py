"""The backward launch table of backward_layers.py, which the dgrad/wgrad fuzz of test_gpu_backward_fuzz.py runs, against
the library, for every frame count, width and depth: one entry per conv in the library's conv order with that conv's
shape; data-gradient launches that cover each conv's input rows exactly once and need the transposed weights the
library packs; plane ranges that lie inside their tensors, whose sizes are the library's workspace tensors.  If the
library's layout changes and the table does not, the fuzz would test launches the backbone no longer makes: this
fails instead."""
import pytest

from backward_layers import backbone_layers, spec
from oracle import arch_oracle as A

B, H, W = 2, 36, 52          # a training batch for the workspace sizes (full resolution; the backbone runs at half)


def _align(v, a):
    return (v + a - 1) // a * a


def _layers(n, g0, d, recompute):
    """Every choice is forced: spec() would fail drawing from rnd = None."""
    return [spec(kind, None, g0, d, recompute=recompute, **force) for kind, force in backbone_layers(n, g0, d)]


def _ws_bytes(planes):
    """The library's forward workspace (backbone_ws): P8 tensors at half resolution, then u at full resolution."""
    off = 0
    for p in planes:
        off = _align(off + B * p * (H // 2) * (W // 2) * 16, 256)
    return _align(off + B * 8 * H * W * 16, 256)


@pytest.mark.parametrize("recompute", [False, True])
@pytest.mark.parametrize("g0", [64, 96])
@pytest.mark.parametrize("n", [2, 3, 5])
def test_backward_table_is_the_librarys(n, g0, recompute):
    from bin_b200 import _lib
    L = _lib.lib()
    for d in range(1, 13):
        a = _lib.backbone_arch(n, g0, d)
        layers = _layers(n, g0, d, recompute)
        weights = [shape for name, shape in A.backbone_param_shapes(n, g0, d) if name.endswith("weight")]
        assert [(s["cout"], s["cin"], s["k"], s["k"]) for s in layers] == weights, (n, g0, d)
        assert len(layers) == L.bin_backbone_nconv(a) == 5 * d + 6, (n, g0, d)

        packed_t = 0
        for idx, s in enumerate(layers):
            where = (n, g0, d, idx, s.get("tag", ""))
            cin, cout = s["cin"], s["cout"]
            # input segments: 4-plane multiples that hold the Cin channels and at most one partial 32-channel block
            planes = [np_ for _, _, np_ in s["x"]]
            assert all(p % 4 == 0 and p > 0 for p in planes) and cin <= 8 * sum(planes) < cin + 32, where
            for total, p0, np_ in s["x"]:
                assert 0 <= p0 and p0 + np_ <= total, where
            dy_total, dy_p0 = s["dy"]
            dy_np = (cout + 31) // 32 * 4
            assert 0 <= dy_p0 and dy_p0 + dy_np <= dy_total, where
            # data gradients: row ranges in ascending order that partition [0, cin)
            row = 0
            for dg in s["dgrad"]:
                assert dg["row0"] == row and dg["nrows"] > 0, where
                row += dg["nrows"]
                total, p0, store = dg["out"]
                assert dg["nrows"] <= 8 * store <= _align(dg["nrows"], 32), where
                if total is None:               # in place in the dY tensor: clear of the dY planes the launch reads
                    total = dy_total
                    assert p0 + store <= dy_p0 or dy_p0 + dy_np <= p0, where
                assert 0 <= p0 and p0 + store <= total, where
                packed_t = _align(packed_t + _align(dg["nrows"], 96) * _align(cout, 32) * s["k"] ** 2 * 2, 256)
            assert row == cin, where
        # the transposed-weight blob holds exactly these launches' weights (then GFF.0's zero bias, up to 1152 rows)
        assert L.bin_backbone_packed_t_bytes(a) == _align(packed_t + 1152 * 4, 256), (n, g0, d)

        # tensor sizes: x0, f1, f2, cat, growth maps, t1, t2 as the table has them give the library's forward workspace
        # (the saving layout, or the inference layout that the recomputing backward rebuilds the growth maps in)
        sfe1, sfe2, rdb0, lff, gff0, gff1, up0 = (layers[j] for j in (0, 1, 2, 2 + 5 * d - 1, -4, -3, -2))
        tensors = [sfe1["x"][0][0], sfe2["x"][0][0], rdb0["x"][0][0], gff0["x"][0][0], lff["x"][1][0], gff1["x"][0][0],
                   up0["x"][0][0]]
        ws = L.bin_backbone_workspace_bytes(a, B, H, W) if recompute else L.bin_backbone_train_workspace_bytes(a, B, H, W)
        assert ws == _ws_bytes(tensors), (n, g0, d, tensors)
        # every RDB reads its input from f2 or cat and its growth maps from that one tensor; d cat is cat's size
        for s in layers[2:2 + 5 * d]:
            assert s["x"][0][0] in (tensors[2], tensors[3]) and all(t == tensors[4] for t, _, _ in s["x"][1:]), s["tag"]
            assert s["cout"] == 32 and s["dy"][0] == 16 or s["dy"][0] == tensors[3], s["tag"]
