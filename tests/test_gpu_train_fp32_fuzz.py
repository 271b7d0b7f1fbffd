"""fp32 kernels of the training step against fp64, per element, with bars derived from the arithmetic.

Part 1 holds bin_convlstm_bwd_ex (atomic and BIN_DETERMINISTIC sums) to fp64, split at its kernel boundaries: the gates
kernel (pass 1: d gates, dc_prev), the weight kernel (pass 2: dw, db) and the input kernel (pass 3: dx, dh_prev), each
first against the exact sum of the kernel's own fp32 terms and then against fp64 truth.  Shapes cover H or W of 1, the
weight kernel's 592-block cap, grid-stride loops that iterate (also in a child that sees 8 SMs), saturated gates, a
forget gate near 0, dh-only and dc-only cotangents and every subset of NULL outputs.  Part 2 holds the pixel loss
(bin_pixel_loss_fwd_ex, bin_pixel_loss_bwd) to fp64 for all three kinds, 1 to 17 pairs and sizes that iterate both
grid-stride loops.  Part 3 checks bin_grad_scale's contract exactly, and the backbone backward that calls it with
non-finite, zero and misaligned cotangents.

Bars (u = 2^-24, the fp32 unit roundoff; gamma_n = n u / (1 - n u)):
  ConvLSTM gates      each gate sum is the bias plus n FMAs (n = 54 with the state, 27 without), and the forget gate adds
                      the forget bias 1: e_k <= K u G_k, K = n + 2, G_k = |b_k| + sum |w||in| (+ 1 for f).
  ConvLSTM pass 1     a first-order running error bound, evaluated in fp64 along the kernel's own expression: every value
                      v carries E_v; a gate error e moves sigmoid by s(1-s) e and tanh by (1-t^2) e; sigmoid
                      1/(1+expf(-g)) adds T_SIG u s (expf <= 2 ulp = 4u of its result, the add and the divide one u
                      each), tanhf adds T_TANH u |t| (<= 2 ulp); a product or quotient adds one u of its magnitude per
                      rounding, a sum one u of the sum of its terms' magnitudes, and 1 - s, 1 - t^2 carry E_s, 2|t| E_t.
                      This is sum_k |d out / d g_k| e_k plus the elementwise chain's roundings with every subtraction
                      taken as an addition of magnitudes (1 - s: E_s + u(1 - s), not u(1 - s): the cancellation near a
                      saturated gate).  FMA contraction only removes roundings.  bar1 = SLACK * E: SLACK = 2 covers the
                      dropped products of two errors, below 1e-3 of E at the gate sums used (|g| < 80).
  ConvLSTM pass 3     dx / dh_prev: up to 108 FMAs from 0, so gamma_108 sum |w||dgates| against the exact sum of the
                      kernel's own dgates; against truth that plus sum |w| bar1(dgates).
  ConvLSTM pass 2     dw / db: L pixels per lane, a 5-level shuffle tree and P block partials (atomics or the ordered
                      reduce): gamma_n sum |terms|, n = L + 10 + P, against the kernel's own terms; against truth that plus
                      sum bar1(dgates) |in|.
  loss backward       L1 is exact (g = upstream / npairs, times +-1 or 0).  L2: d (u), upstream / npairs (u), g * 2d (u):
                      gamma_3 |ref|.  Charbonnier d / sqrtf(d^2 + eps): d (u), d^2 (u), + eps (u), sqrtf (half the
                      argument's 4u, plus u), the divide (u) make 5u; g = upstream / npairs * (1 / n) three more, g * t
                      one: gamma_9 |ref|.
  loss forward        against fp64 of the kernel's fp32 differences: each term rounds at most twice (2u), then every
                      term passes through at most T adds in its thread (the loop trip count), 5 shuffle levels, 8 warp
                      partials and P block partials (atomics) or ceil(P/32) + 5 (the ordered reduce), and the
                      Charbonnier mean divides once: gamma_(T + 5 + 8 + P + 5 + 3) sum |terms|.
  loss scale          exact: scale is a power of two with scale * max <= target < 2 scale max.
"""
import ctypes as C
import math
import os
import statistics
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda"
NAN = float("nan")
SENTINEL = -1234.5
U = 2.0 ** -24
K_GATE = {True: 56.0, False: 29.0}      # FMAs of one gate sum (54 / 27) + 2
T_SIG = 6.0
T_TANH = 4.0
SLACK = 2.0
TAPS_DX = 108                           # 12 gates x 9 taps per dx / dh_prev element
LOSS_EPS = float(np.float32(1e-6))      # the eps the kernel sees
RATIOS = {}                             # label -> [worst error / bar of each case]


def gamma(n):
    return n * U / (1 - n * U)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for key in sorted(RATIOS):
        r = sorted(RATIOS[key])
        print(f"[fp32 fuzz] {key:<20} cases {len(r):3d}  worst err/bar {r[-1]:.3g}  median {statistics.median(r):.3g}")


def _record(label, ratio):
    RATIOS.setdefault(label, []).append(ratio)


def _bits(t):
    return t.contiguous().view(torch.int32)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _ratio(got, ref, bar, where):
    """Worst |got - ref| / bar; where bar is 0 the kernel must be exact."""
    if got.numel() == 0:                  # e.g. n = 1 with its one element masked out as the NaN target
        return 0.0
    got = got.double()
    assert torch.isfinite(got).all(), ("non-finite output", where)
    err = (got - ref).abs()
    r = torch.where(bar > 0, err / bar.clamp_min(1e-300), torch.where(err > 0, math.inf, 0.0))
    return r.max().item()


def _check(label, got, ref, bar, where):
    r = _ratio(got, ref, bar, where)
    _record(label, r)
    assert r <= 1.0, (label, where, r)
    return r


# --------------------------------------------------------------------------------------------------------------------
# part 1: the ConvLSTM backward
# --------------------------------------------------------------------------------------------------------------------
def _lstm_inputs(B, H, W, state, cot, seed):
    """fp32 inputs.  Weights N(0, 0.8^2) on inputs in [0, 3) give gate sums that spread over about +-40, so many gates
    are saturated (|g| > 10); the biases of input gate 1 (+12) and forget gate 6 (-14) push those two further, so some
    forget gates are near 0.  No gate sum reaches 80 (expf(80) and its sigmoid stay normal)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.rand((B, 3, H, W), generator=g, device=DEV) * 3
    w = torch.randn((12, 6, 3, 3), generator=g, device=DEV) * 0.8
    b = torch.randn((12,), generator=g, device=DEV) + torch.tensor([0, 12] + [0] * 4 + [-14] + [0] * 5, device=DEV)
    cp = torch.randn((B, 3, H, W), generator=g, device=DEV) * 4 if state else None
    hp = torch.rand((B, 3, H, W), generator=g, device=DEV) * 2 - 1 if state else None
    dh = torch.randn((B, 3, H, W), generator=g, device=DEV) if cot in ("both", "dh") else None
    dc = torch.randn((B, 3, H, W), generator=g, device=DEV) if cot in ("both", "dc") else None
    return x, cp, hp, w, b, dh, dc


def _lstm_abi(x, cp, hp, w, b, dh, dc, flags, want=("dx", "dcp", "dhp", "dw", "db")):
    """bin_convlstm_bwd_ex.  Every output buffer starts as SENTINEL, except requested dw / db, which start at 0 (the
    call accumulates); an output not in `want` is passed as NULL.  Returns (outputs by name, dgates)."""
    from bin_b200 import _lib
    L = _lib.lib()
    B, _, H, W = x.shape
    out = {k: torch.full_like(x, SENTINEL) for k in ("dx", "dcp", "dhp")}
    out["dw"] = torch.zeros_like(w) if "dw" in want else torch.full_like(w, SENTINEL)
    out["db"] = torch.zeros_like(b) if "db" in want else torch.full_like(b, SENTINEL)
    dgates = torch.full((B, 12, H, W), SENTINEL, device=DEV)
    scratch = torch.empty(L.bin_convlstm_bwd_scratch_bytes(B, H, W), dtype=torch.uint8, device=DEV)
    P = lambda t: None if t is None else t.data_ptr()
    O = lambda k: out[k].data_ptr() if k in want else None
    _lib.check(L.bin_convlstm_bwd_ex(x.data_ptr(), P(cp), P(hp), w.data_ptr(), b.data_ptr(), P(dh), P(dc),
                                     dgates.data_ptr(), O("dx"), O("dcp"), O("dhp"), O("dw"), O("db"), B, H, W, flags,
                                     scratch.data_ptr(), scratch.numel(), _stream()))
    torch.cuda.synchronize()
    return out, dgates


def _pass1_ref(x, cp, hp, w, b, dh, dc):
    """fp64 d gates (B,12,H,W) and dc_prev from the fp32 inputs, and their bars bar1 (see the module docstring)."""
    state = cp is not None
    z = torch.zeros(x.shape, dtype=torch.float64, device=DEV)
    c0 = cp.double() if state else z
    xh = torch.cat((x.double(), hp.double() if state else z), 1)
    g = F.conv2d(xh, w.double(), b.double(), padding=1)
    G = F.conv2d(xh.abs(), w.double().abs(), b.double().abs(), padding=1)
    K = K_GATE[state]
    gi, gj, gf, go = g.chunk(4, 1)
    Gi, Gj, Gf, Go = G.chunk(4, 1)
    gf = gf + 1.0
    ei, ej, ef, eo = K * U * Gi, K * U * Gj, K * U * (Gf + 1.0), K * U * Go
    dhv = dh.double() if dh is not None else z
    dcv = dc.double() if dc is not None else z
    si, tj, sf, so = torch.sigmoid(gi), torch.tanh(gj), torch.sigmoid(gf), torch.sigmoid(go)
    E_si = si * (1 - si) * ei + T_SIG * U * si
    E_tj = (1 - tj * tj) * ej + T_TANH * U * tj.abs()
    E_sf = sf * (1 - sf) * ef + T_SIG * U * sf
    E_so = so * (1 - so) * eo + T_SIG * U * so
    cn = c0 * sf + si * tj
    E_cn = c0.abs() * E_sf + tj.abs() * E_si + si * E_tj + 2 * U * (c0.abs() * sf + si * tj.abs())
    tc = torch.tanh(cn)
    E_tc = (1 - tc * tc) * E_cn + T_TANH * U * tc.abs()
    q = 1 - tc * tc
    E_q = 2 * tc.abs() * E_tc + U * (tc * tc + q)
    p = dhv * so * q
    dct = dcv + p
    E_dct = dhv.abs() * (q * E_so + so * E_q) + 2 * U * p.abs() + U * (dcv.abs() + p.abs())
    ai, af, ao = 1 - si, 1 - sf, 1 - so
    E_ai, E_af, E_ao = E_si + U * ai, E_sf + U * af, E_so + U * ao
    bj = 1 - tj * tj
    E_bj = 2 * tj.abs() * E_tj + U * (tj * tj + bj)
    d_i = dct * tj * si * ai
    d_j = dct * si * bj
    d_f = dct * c0 * sf * af
    d_o = dhv * tc * so * ao
    dcp = dct * sf
    A = dct.abs()
    E_i = (tj.abs() * si * ai * E_dct + A * (si * ai * E_tj + tj.abs() * ai * E_si + tj.abs() * si * E_ai)
           + 3 * U * d_i.abs())
    E_j = si * bj * E_dct + A * (bj * E_si + si * E_bj) + 2 * U * d_j.abs()
    E_f = c0.abs() * sf * af * E_dct + A * c0.abs() * (af * E_sf + sf * E_af) + 3 * U * d_f.abs()
    E_o = dhv.abs() * (so * ao * E_tc + tc.abs() * ao * E_so + tc.abs() * so * E_ao) + 3 * U * d_o.abs()
    E_cp = sf * E_dct + A * E_sf + U * dcp.abs()
    dgates = torch.cat((d_i, d_j, d_f, d_o), 1)
    bar = SLACK * torch.cat((E_i, E_j, E_f, E_o), 1)
    return dgates, bar, dcp, SLACK * E_cp, g, sf


def _inputs6(x, hp):
    return torch.cat((x, torch.zeros_like(x) if hp is None else hp), 1).double()


def _tap_sums(gt, inp):
    """sum_p gt[b,k,p] * inp[b,c,p + tap] for the 9 taps -> (12, 6, 3, 3) (zero padding)."""
    H, W = inp.shape[2], inp.shape[3]
    inp = F.pad(inp, (1, 1, 1, 1))
    out = torch.zeros((12, 6, 9), dtype=torch.float64, device=DEV)
    for t in range(9):
        ky, kx = divmod(t, 3)
        out[:, :, t] = torch.einsum("bkyx,bcyx->kc", gt, inp[:, :, ky:ky + H, kx:kx + W])
    return out.reshape(12, 6, 3, 3)


def _lstm_case(shape, state, flags, cot, seed):
    """One call with every output against fp64; returns the worst err/bar.  Asserts (and records) every check."""
    B, H, W = shape
    where = (shape, state, flags, cot)
    x, cp, hp, w, b, dh, dc = _lstm_inputs(B, H, W, state, cot, seed)
    want = ("dx", "dcp", "dhp", "dw", "db") if state else ("dx", "dw", "db")
    out, dg = _lstm_abi(x, cp, hp, w, b, dh, dc, flags, want)
    ref_g, bar1, ref_cp, bar_cp, gsum, sf = _pass1_ref(x, cp, hp, w, b, dh, dc)
    if B * H * W >= 4000:                                    # the inputs reach the regimes the bars are written for
        assert (gsum.abs() > 10).any() and (sf < 1e-4).any() and gsum.abs().max() < 80, where
    worst = 0.0
    # pass 1
    worst = max(worst, _check("lstm dgates", dg, ref_g, bar1, where))
    if state:
        worst = max(worst, _check("lstm dc_prev", out["dcp"], ref_cp, bar_cp, where))
    else:
        for k in ("dcp", "dhp"):
            assert (out[k] == SENTINEL).all(), (k, where)
    # pass 3: dx, dh_prev
    wd = w.double()
    own = F.conv_transpose2d(dg.double(), wd, padding=1)
    own_abs = F.conv_transpose2d(dg.double().abs(), wd.abs(), padding=1)
    truth = F.conv_transpose2d(ref_g, wd, padding=1)
    prop = F.conv_transpose2d(bar1, wd.abs(), padding=1)
    bar_own = gamma(TAPS_DX) * own_abs
    for name, sl in (("dx", slice(0, 3)), ("dh_prev", slice(3, 6))):
        if name == "dh_prev" and not state:
            continue
        got = out["dx" if name == "dx" else "dhp"]
        worst = max(worst, _check(f"lstm {name} own", got, own[:, sl], bar_own[:, sl], where))
        worst = max(worst, _check(f"lstm {name}", got, truth[:, sl], bar_own[:, sl] + prop[:, sl], where))
    # pass 2: dw, db
    inp = _inputs6(x, hp)
    total = B * H * W
    P = min((total + 31) // 32, 592)
    bar_g = gamma(-(-total // (P * 32)) + 10 + P)
    gd = dg.double()
    ew, aw = _tap_sums(gd, inp), _tap_sums(gd.abs(), inp.abs())
    eb, ab = gd.sum((0, 2, 3)), gd.abs().sum((0, 2, 3))
    tw, pw = _tap_sums(ref_g, inp), _tap_sums(bar1, inp.abs())
    tb, pb = ref_g.sum((0, 2, 3)), bar1.sum((0, 2, 3))
    worst = max(worst, _check("lstm dw own", out["dw"], ew, bar_g * aw, where))
    worst = max(worst, _check("lstm db own", out["db"], eb, bar_g * ab, where))
    worst = max(worst, _check("lstm dw", out["dw"], tw, bar_g * aw + pw, where))
    worst = max(worst, _check("lstm db", out["db"], tb, bar_g * ab + pb, where))
    if not state:
        assert torch.equal(_bits(out["dw"][:, 3:6]), _bits(torch.zeros_like(out["dw"][:, 3:6]))), where
    return worst


LSTM_SHAPES = [(1, 1, 1), (1, 1, 37), (3, 29, 1), (2, 2, 2), (1, 17, 33), (2, 96, 128), (3, 256, 384), (1, 720, 1280)]
COTS = ("both", "dh", "dc")


@pytest.mark.parametrize("flags", [0, 1])
@pytest.mark.parametrize("state", [False, True])
@pytest.mark.parametrize("shape", LSTM_SHAPES)
def test_convlstm_backward_vs_fp64(shape, state, flags):
    idx = LSTM_SHAPES.index(shape)
    if shape == (3, 256, 384):                   # the gates and input kernels' grids (132 SMs x 16 blocks x 128 px) wrap
        assert shape[0] * shape[1] * shape[2] > torch.cuda.get_device_properties(0).multi_processor_count * 16 * 128
    cot = COTS[(idx + state) % 3]
    r = _lstm_case(shape, state, flags, cot, seed=700 + 4 * idx + 2 * state + flags)
    print(f"[fp32 fuzz] convlstm {shape} state={state} flags={flags} cot={cot}: worst err/bar {r:.3g}")


@pytest.mark.parametrize("state", [False, True])
def test_convlstm_null_outputs_keep_bits(state):
    """Every subset of the outputs: each requested one has the bits of the all-outputs call (dw and db in the
    deterministic mode, whose sums have a fixed order), every other buffer keeps its sentinel."""
    names = ("dx", "dcp", "dhp", "dw", "db") if state else ("dx", "dw", "db")
    x, cp, hp, w, b, dh, dc = _lstm_inputs(2, 17, 33, state, "both", seed=90 + state)
    for flags in (0, 1):
        full, _ = _lstm_abi(x, cp, hp, w, b, dh, dc, flags, names)
        for mask in range(1 << len(names)):
            want = tuple(n for i, n in enumerate(names) if mask >> i & 1)
            out, _ = _lstm_abi(x, cp, hp, w, b, dh, dc, flags, want)
            for n in ("dx", "dcp", "dhp", "dw", "db"):
                if n in want:
                    if flags or n not in ("dw", "db"):
                        assert torch.equal(_bits(out[n]), _bits(full[n])), (flags, want, n)
                else:
                    assert (out[n] == SENTINEL).all(), (flags, want, n)


_CHILD = r"""
import sys
sys.path[:0] = [%r, %r]
import test_gpu_train_fp32_fuzz as T
worst = 0.0
for state in (False, True):
    for flags in (0, 1):
        worst = max(worst, T._lstm_case((2, 96, 128), state, flags, "both", seed=800 + 2 * state + flags))
print("LSTM", worst)
T._grad_scale_positions()
print("SCALE ok")
"""


def test_small_sm_count_child():
    """With BIN_B200_MAX_SMS=8 the gates and input kernels run 128 blocks of 128 px, so at 2 x 96 x 128 px their
    grid-stride loops iterate, and so does the loss-scale maximum over 2.1M floats."""
    env = dict(os.environ, BIN_B200_MAX_SMS="8")
    r = subprocess.run([sys.executable, "-c", _CHILD % (ROOT, os.path.join(ROOT, "tests"))], env=env,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    lines = dict(line.split(" ", 1) for line in r.stdout.strip().splitlines() if line[:5] in ("LSTM ", "SCALE"))
    assert float(lines["LSTM"]) <= 1.0 and lines["SCALE"] == "ok", r.stdout[-2000:]
    _record("lstm 8 SMs", float(lines["LSTM"]))


# --------------------------------------------------------------------------------------------------------------------
# part 2: the pixel loss
# --------------------------------------------------------------------------------------------------------------------
def _ptrs(ts):
    return (C.c_void_p * len(ts))(*[None if t is None else t.data_ptr() for t in ts])


def _loss_fwd(a, b, n, kind, flags):
    from bin_b200 import _lib
    L = _lib.lib()
    npairs = len(a)
    pair = torch.full((npairs,), SENTINEL, device=DEV)
    nbytes = L.bin_pixel_loss_scratch_bytes(npairs, n)
    scratch = torch.empty(max(nbytes, 4), dtype=torch.uint8, device=DEV)
    _lib.check(L.bin_pixel_loss_fwd_ex(_ptrs(a), _ptrs(b), npairs, n, kind, LOSS_EPS, pair.data_ptr(), flags,
                                       scratch.data_ptr(), nbytes, _stream()))
    torch.cuda.synchronize()
    return pair


def _loss_bwd(a, b, n, kind, up, db_mode):
    """bin_pixel_loss_bwd; db_mode 0: every db, 1: db_host NULL, 2: every other db entry NULL.  Returns (da, db) with
    None where no db was passed (the buffers still exist and must keep the sentinel)."""
    from bin_b200 import _lib
    npairs = len(a)
    da = [torch.full((n,), SENTINEL, device=DEV) for _ in range(npairs)]
    db = [torch.full((n,), SENTINEL, device=DEV) for _ in range(npairs)]
    passed = [db_mode == 0 or (db_mode == 2 and k % 2 == 0) for k in range(npairs)]
    upt = torch.tensor([up], dtype=torch.float32, device=DEV)
    dbp = None if db_mode == 1 else _ptrs([t if p else None for t, p in zip(db, passed)])
    _lib.check(_lib.lib().bin_pixel_loss_bwd(_ptrs(a), _ptrs(b), _ptrs(da), dbp, npairs, n, kind, LOSS_EPS,
                                              upt.data_ptr(), _stream()))
    torch.cuda.synchronize()
    return da, db, passed


def _fwd_blocks(n):
    return min(-(-n // 4096), 256)


LOSS_N = [1, 3, 4097, 256 * 4096 + 1, 2 * 512 * 2048 + 3]
KIND_NAMES = ("l1", "l2", "cb")


@pytest.mark.parametrize("n", LOSS_N)
@pytest.mark.parametrize("kind", [0, 1, 2])
def test_pixel_loss_vs_fp64(kind, n):
    kn = KIND_NAMES[kind]
    for npairs in (1, 3, 17):
        gen = torch.Generator(device=DEV).manual_seed(1000 * kind + npairs + n % 997)
        a = [torch.rand((n,), generator=gen, device=DEV) for _ in range(npairs)]
        b = [torch.rand((n,), generator=gen, device=DEV) for _ in range(npairs)]
        for k in range(npairs):                          # d == 0 exactly at every 7th element
            b[k][::7] = a[k][::7]
        if npairs > 1:                                   # a cycle term: the last pair's target is pair 0's prediction
            b[-1] = a[0]
        # ---- forward, both modes, per pair against fp64 of the kernel's fp32 differences
        P = _fwd_blocks(n)
        T = -(-n // (P * 256))
        bar_rel = gamma(T + 5 + 8 + P + 5 + 3)
        for flags in (0, 1):
            got = _loss_fwd(a, b, n, kind, flags).double()
            for k in range(npairs):
                d = (a[k] - b[k]).double()
                t = d.abs() if kind == 0 else (d * d if kind == 1 else torch.sqrt(d * d + LOSS_EPS))
                ref = t.sum() / (n if kind == 2 else 1)
                _check(f"loss fwd {kn}", got[k:k + 1], ref.view(1), (bar_rel * ref).view(1), (kn, n, npairs, flags, k))
        # ---- backward: NaN in pair 0's target, upstream 0.37 / 2^-20 / 1
        b0 = b[0].clone()
        b0[n // 2] = NAN
        bb = [b0] + b[1:]
        nanmask = torch.zeros(n, dtype=torch.bool, device=DEV)
        nanmask[n // 2] = True
        up = float(np.float32((0.37, 2.0 ** -20, 1.0)[(n + npairs) % 3]))       # the upstream the kernel reads
        db_mode = (kind + npairs) % 3
        da, db, passed = _loss_bwd(a, bb, n, kind, up, db_mode)
        g32 = torch.tensor([up], dtype=torch.float32, device=DEV) / torch.tensor([float(npairs)], device=DEV)
        for k in range(npairs):
            where = (kn, n, npairs, k, up, db_mode)
            d32 = a[k] - bb[k]
            if kind == 0:                                # exact: g * (+-1 or 0), and 0 where the target is NaN
                t = torch.where(d32 > 0, 1.0, torch.where(d32 < 0, -1.0, 0.0))
                assert torch.equal(_bits(da[k]), _bits(g32 * t)), where
                if passed[k]:
                    assert torch.equal(_bits(db[k]), _bits(-g32 * t)), where
            else:
                d = (a[k].double() - bb[k].double())
                g64 = up / npairs
                tr = 2 * d if kind == 1 else d / torch.sqrt(d * d + LOSS_EPS) / n
                ref = g64 * tr
                bar = gamma(3 if kind == 1 else 9) * ref.abs()
                nan0 = nanmask if k == 0 else torch.zeros_like(nanmask)
                assert torch.isnan(da[k][nan0]).all(), where
                _check(f"loss bwd {kn}", da[k][~nan0], ref[~nan0], bar[~nan0], where)
                if passed[k]:
                    assert torch.isnan(db[k][nan0]).all(), where
                    _check(f"loss bwd {kn}", db[k][~nan0], -ref[~nan0], bar[~nan0], where)
            if not passed[k]:
                assert (db[k] == SENTINEL).all(), where


# --------------------------------------------------------------------------------------------------------------------
# part 3: the device loss scale and the backbone backward that uses it
# --------------------------------------------------------------------------------------------------------------------
SCALE_TARGETS = (1.0, 3.0, 1024.0, 2048.0)


def _grad_scale(ts, numel, target):
    from bin_b200 import _lib
    out = torch.empty(2, device=DEV)
    _lib.check(_lib.lib().bin_grad_scale(_ptrs(ts), len(ts), numel, target, out.data_ptr(), out.data_ptr() + 4,
                                         _stream()))
    return out[0].item()


def _contract(s, gmax, target):
    """scale is a positive power of two with s * max <= target < 2 s max, in exact arithmetic (fp64 holds the
    products of a power of two and an fp32 value exactly)."""
    return s > 0 and math.frexp(s)[0] == 0.5 and s * gmax <= target < 2 * s * gmax


def test_grad_scale_exact_contract():
    """Maxima 2^j (1 + m 2^-23), m in -4..4, over every j that keeps the scale a normal float (and the maximum above
    the 1e-30 clamp), at four targets; each maximum sits in a row of four floats whose other entries are smaller."""
    from bin_b200 import _lib
    L = _lib.lib()
    js, ms = range(-99, 126), range(-4, 5)
    maxima = np.array([np.float32(2.0 ** j * (1 + m * 2.0 ** -23)) for j in js for m in ms], dtype=np.float32)
    rows = np.stack([maxima * 0.5, -maxima, maxima * 0.25, np.zeros_like(maxima)], 1).astype(np.float32)
    rows[1::2, 1] *= -1                                          # the maximum is negative in half the rows
    g = torch.from_numpy(rows).to(DEV).contiguous()
    bad = []
    for target in SCALE_TARGETS:
        scales = torch.full((len(maxima),), NAN, device=DEV)
        tmp = torch.empty((len(maxima),), dtype=torch.int32, device=DEV)
        for r in range(len(maxima)):
            _lib.check(L.bin_grad_scale((C.c_void_p * 1)(g.data_ptr() + 16 * r), 1, 4, target,
                                        scales.data_ptr() + 4 * r, tmp.data_ptr() + 4 * r, _stream()))
        s = scales.cpu().numpy().astype(np.float64)
        for r, (gm, sc) in enumerate(zip(maxima.astype(np.float64), s)):
            if not _contract(float(sc), float(gm), target):
                bad.append((target, js[r // len(ms)], ms[r % len(ms)], float(gm), float(sc)))
    assert not bad, (len(bad), bad[:12])


def _grad_scale_positions():
    """Where the maximum sits: call n-1 of 6, the tail when numel % 4 is 1..3, the last float4 of a grid-stride loop,
    negative; plus -0.0, all zeros (the 1e-30 clamp), a NaN (ignored) and an inf (scale 0)."""
    gen = torch.Generator(device=DEV).manual_seed(17)
    vmax = float(np.float32(8.0 * (1 + 3 * 2.0 ** -23)))

    def case(ncalls, numel, call, idx, sign=1.0):
        ts = [(torch.rand((numel,), generator=gen, device=DEV) * 2 - 1) * 4 for _ in range(ncalls)]
        ts[call][idx] = sign * vmax
        for target in SCALE_TARGETS:
            s = _grad_scale(ts, numel, target)
            assert _contract(s, vmax, target), (ncalls, numel, call, idx, sign, target, s)

    case(6, 1000, 5, 999)
    case(6, 4099, 5, 17, -1.0)
    for r in (1, 2, 3):
        for call in (0, 2):
            case(3, 4 * 250 + r, call, 4 * 250 + r - 1)
    big = 2 * 132 * 16 * 256 * 4 + 8                              # more float4s than the absmax grid has threads
    case(1, big, 0, big - 1)
    case(2, big, 1, big - 4, -1.0)
    case(1, big + 3, 0, big + 2)
    clamp = float(np.float32(1e-30))
    for fill in (0.0, -0.0):
        t = torch.full((1001,), fill, device=DEV)
        for target in SCALE_TARGETS:
            s = _grad_scale([t], 1001, target)
            assert math.isfinite(s) and _contract(s, clamp, target), (fill, target, s)
    t = torch.rand((4097,), generator=gen, device=DEV)
    t[100] = vmax
    t[4096] = NAN
    t[7] = NAN
    assert _contract(_grad_scale([t], 4097, 2048.0), vmax, 2048.0)
    t[4000] = -math.inf
    assert _grad_scale([t], 4097, 2048.0) == 0.0


def test_grad_scale_where_the_maximum_sits():
    _grad_scale_positions()


@pytest.fixture
def det():
    prev = (torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled(),
            torch.utils.deterministic.fill_uninitialized_memory)
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(prev[0], warn_only=prev[1])
    torch.utils.deterministic.fill_uninitialized_memory = prev[2]


@pytest.fixture(scope="module")
def backbone():
    from bin_b200 import rdn
    from oracle import bin_oracle as O
    net = rdn.bin_stage4_lstm()
    net.load_state_dict(O.synth_state_dict(0), strict=True)
    net = net.cuda().train()
    frames = [f.cuda() for f in O.synth_frames(2, 1, 32, 64, seed=61, smooth=True)]
    return net.model.model1_1, frames


def _stage_grads(model, frames, cot):
    from bin_b200.autograd import backbone_stage
    for p in model.parameters():
        p.grad = None
    fr = [f.clone().requires_grad_(True) for f in frames]
    (out,) = backbone_stage(model, [fr])
    torch.autograd.backward([out], [cot])
    torch.cuda.synchronize()
    return [p.grad.clone() for p in model.parameters()] + [f.grad.clone() for f in fr]


@pytest.mark.parametrize("value", [math.inf, NAN])
def test_nonfinite_cotangent_leaves_nonfinite_gradients(backbone, value):
    """An inf maximum gives scale 0 and a NaN is skipped by the maximum; either way the parameter gradients must come
    out non-finite, which is what makes the optimizer's guard skip the step."""
    model, frames = backbone
    cot = torch.rand_like(frames[0]) - 0.5
    cot[0, 1, 13, 40] = value
    grads = _stage_grads(model, frames, cot)[:-2]
    bad = sum(1 for t in grads if not torch.isfinite(t).all())
    assert bad > 0, value


def test_zero_cotangent_gives_zero_gradients(backbone):
    model, frames = backbone
    for fill in (0.0, -0.0):
        grads = _stage_grads(model, frames, torch.full_like(frames[0], fill))
        assert all(torch.isfinite(t).all() and (t == 0).all() for t in grads), fill


def test_misaligned_cotangent(det, backbone):
    """A cotangent that is a contiguous view 4 bytes into its storage gives the gradients of an aligned copy, bit for
    bit (the loss scale reads float4s, so the backward copies it)."""
    model, frames = backbone
    base = torch.rand(frames[0].numel() + 1, device=DEV) - 0.5
    cot = base[1:].view_as(frames[0])
    assert cot.is_contiguous() and cot.data_ptr() % 16 == 4
    got = _stage_grads(model, frames, cot)
    ref = _stage_grads(model, frames, cot.clone())
    assert all(torch.equal(a, b) for a, b in zip(got, ref))
