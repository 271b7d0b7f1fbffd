"""GPU checks of bin_png_encode_u8 and bin_b200.png: every file passes the strict reader, inflates to the payload
cv2.imwrite writes and gives the pixels back; sizes against cv2's (zlib level 1, Z_RLE); the cv2 fixture; the same
bytes across repeats, streams, batch positions, batch sizes and SM counts; guard bytes; test.py's write path from a
window's output; and the refusals."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import bin_oracle as O
from oracle import png_oracle as P

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SHAPES = [(1, 1), (1, 2), (2, 1), (7, 9), (37, 53), (64, 128), (720, 1280), (768, 1344), (2160, 3840)]
KINDS = ["noise", "flat", "smooth", "natural", "stripes", "runs", "long_run"]


def _from_sub(sub):
    h, n = sub.shape
    rgb = (np.cumsum(sub.reshape(h, n // 3, 3).astype(np.uint64), axis=1) % 256).astype(np.uint8)
    return np.ascontiguousarray(rgb[:, :, ::-1])


def make_image(kind, h, w, seed=0):
    rng = np.random.default_rng(seed)
    if kind == "noise":
        return rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8)
    if kind == "flat":
        return np.full((h, w, 3), (30, 120, 200), np.uint8)
    if kind in ("smooth", "natural"):                # natural: blurred noise plus Gaussian noise (test_gpu_metrics._pair)
        from scipy.ndimage import gaussian_filter
        z = gaussian_filter(rng.standard_normal((h, w, 3)), sigma=(4.0, 4.0, 0.0))
        a = np.clip(np.round((z - z.min()) / max(z.max() - z.min(), 1e-9) * 235 + 10), 0, 255).astype(np.int32)
        if kind == "natural":
            a = a + rng.normal(0, 4, size=a.shape).round().astype(np.int32)
        return np.clip(a, 0, 255).astype(np.uint8)
    if kind == "stripes":
        x = np.arange(w)
        return np.repeat(np.where((x // 5) % 2, 220, 17).astype(np.uint8)[None, :, None], h, 0).repeat(3, 2)
    if kind == "runs":                               # Sub bytes with runs of 257..261 repeats wherever a row has room
        sub = rng.integers(1, 256, size=(h, 3 * w), dtype=np.uint8)
        for y in range(h):
            r = 257 + y % 5
            if 3 * w > r + 2:
                s = int(rng.integers(1, 3 * w - r - 1))
                sub[y, s:s + r + 1] = 0
        return _from_sub(sub)
    if kind == "long_run":                           # every payload byte is 1: one run across all segments
        return _from_sub(np.ones((h, 3 * w), np.uint8))
    raise ValueError(kind)


def _lib():
    from bin_b200._lib import lib
    return lib()


def _check_file(data, img):
    raw, pix = P.parse_png(data)
    assert raw == P.payload(img)
    assert np.array_equal(pix, img)


@pytest.mark.parametrize("h,w", SHAPES)
def test_cases_round_trip_and_size(h, w):
    from bin_b200.png import encode_png
    worst = int(_lib().bin_png_max_bytes(h, w))
    ratios = []
    for i, kind in enumerate(KINDS):
        img = make_image(kind, h, w, seed=100 + i)
        data = encode_png([torch.from_numpy(img).cuda()])[0]
        _check_file(data, img)
        ref = P.cv2_like_size(img)
        ratios.append(f"{kind} {len(data) / ref:.4f}")
        assert len(data) <= worst
        assert len(data) <= 1.01 * ref + 16384, (kind, len(data), ref)
        if (h, w) in ((720, 1280), (768, 1344)) and kind in ("natural", "noise"):
            assert len(data) <= 1.01 * ref, (kind, len(data), ref)
    print(f"PNG size / cv2 size at {h}x{w}: " + ", ".join(ratios))


def test_golden_fixture(golden_dir, tmp_path):
    from bin_b200.png import encode_png, imwrite
    g = np.load(os.path.join(golden_dir, "png.npz"))
    try:
        import cv2
    except ImportError:
        cv2 = None
    for name in g["names"]:
        img, cv2_file = g[f"{name}_img"], g[f"{name}_png"].tobytes()
        data = encode_png([torch.from_numpy(img).cuda()])[0]
        raw, pix = P.parse_png(data)
        assert raw == P.parse_png(cv2_file)[0], name
        assert np.array_equal(pix, img), name
        print(f"{name}: {len(data)} bytes, cv2 fixture {len(cv2_file)}")
        if cv2 is not None:
            path = str(tmp_path / f"{name}.png")
            assert imwrite(path, img)
            assert np.array_equal(cv2.imread(path, cv2.IMREAD_UNCHANGED), img), name
            live = len(cv2.imencode(".png", img)[1])
            assert len(data) <= 1.01 * live + 16384, (name, len(data), live)


def _hashes(files):
    import hashlib
    return [hashlib.sha256(f).hexdigest() for f in files]


def test_same_bytes_across_repeats_streams_positions_and_batch_sizes():
    from bin_b200.png import encode_png
    h, w = 96, 160
    imgs = [torch.from_numpy(make_image(KINDS[i % len(KINDS)], h, w, seed=7 + i)).cuda() for i in range(16)]
    one = [encode_png([x])[0] for x in imgs]
    for x, f in zip(imgs, one):
        _check_file(f, x.cpu().numpy())
    assert encode_png(imgs) == one                                  # n = 16
    assert encode_png(imgs[5:8]) == one[5:8]                        # n = 3
    rev = encode_png(imgs[::-1])
    assert rev == one[::-1]                                         # other batch positions
    for _ in range(3):
        assert encode_png(imgs[:3]) == one[:3]
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        got = encode_png(imgs[2:5])
    assert got == one[2:5]
    many = encode_png(imgs + imgs[:3])                              # more than one launch sequence
    assert many == one + one[:3]
    big = torch.from_numpy(make_image("natural", 720, 1280, seed=3)).cuda()
    a = encode_png([big, big, big])
    assert a[0] == a[1] == a[2] == encode_png([big])[0]


_CHILD = r"""
import hashlib, sys
sys.path.insert(0, %r)
import torch
from bin_b200.png import encode_png
sys.path.insert(0, %r)
from test_gpu_png import make_image
imgs = [torch.from_numpy(make_image(k, 720, 1280, seed=11)).cuda() for k in ("natural", "noise", "long_run")]
imgs.append(torch.from_numpy(make_image("smooth", 2160, 3840, seed=12)).cuda())
files = encode_png(imgs[:3]) + encode_png(imgs[3:])
print("PNG", hashlib.sha256(b"".join(files)).hexdigest())
"""


def test_results_do_not_depend_on_the_sm_count():
    got = {}
    for tag in ("all", "114", "66"):
        env = {k: v for k, v in os.environ.items() if k != "BIN_B200_MAX_SMS"}
        if tag != "all":
            env["BIN_B200_MAX_SMS"] = tag
        r = subprocess.run([sys.executable, "-c", _CHILD % (ROOT, os.path.join(ROOT, "tests"))], env=env,
                           capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, (tag, r.stderr[-3000:])
        got[tag] = [ln for ln in r.stdout.splitlines() if ln.startswith("PNG ")]
        print("SMS", tag, got[tag])
    assert len({tuple(v) for v in got.values()}) == 1 and got["all"], got


def test_guard_bytes():
    import ctypes as C
    L = _lib()
    h, w, n, guard = 53, 37, 3, 4096
    stride = int(L.bin_png_max_bytes(h, w)) + 5                  # unaligned stride
    imgs_np = [make_image(k, h, w, seed=3) for k in ("noise", "runs", "flat")]
    src = torch.randint(0, 256, (guard + n * h * w * 3 + guard,), dtype=torch.uint8, device="cuda")
    for i, im in enumerate(imgs_np):
        src[guard + i * h * w * 3: guard + (i + 1) * h * w * 3] = torch.from_numpy(im.reshape(-1)).cuda()
    src0 = src.clone()
    out = torch.randint(0, 256, (guard + n * stride + guard,), dtype=torch.uint8, device="cuda")
    out0 = out.clone()
    sizes = torch.full((n + 2,), -7, dtype=torch.int64, device="cuda")
    ws = torch.empty(int(L.bin_png_workspace_bytes(n, h, w)), dtype=torch.uint8, device="cuda")
    ptrs = (C.c_void_p * n)(*[src.data_ptr() + guard + i * h * w * 3 for i in range(n)])
    rc = L.bin_png_encode_u8(ptrs, n, h, w, out.data_ptr() + guard, stride, sizes.data_ptr() + 8, ws.data_ptr(),
                             ws.numel(), torch.cuda.current_stream().cuda_stream)
    assert rc == 0, L.bin_last_error()
    torch.cuda.synchronize()
    assert torch.equal(src, src0)
    assert torch.equal(out[:guard], out0[:guard]) and torch.equal(out[guard + n * stride:], out0[guard + n * stride:])
    sz = sizes.cpu().tolist()
    assert sz[0] == -7 and sz[-1] == -7
    o = out.cpu().numpy()
    for i, im in enumerate(imgs_np):
        base = guard + i * stride
        _check_file(o[base:base + sz[1 + i]].tobytes(), im)
        assert np.array_equal(o[base + sz[1 + i]:base + stride], out0.cpu().numpy()[base + sz[1 + i]:base + stride])


def test_window_output_written_like_test_py(tmp_path):
    from bin_b200 import rdn
    from bin_b200.png import encode_png, encode_png_async, imwrite
    from bin_b200.streaming import tensor2img_u8, test_py_padding
    h, w = 120, 180
    pl, pr, pt, pb = test_py_padding(h, w)
    net = rdn.bin_stage4_lstm()
    net.load_state_dict(O.synth_state_dict(0), strict=True)
    net = net.cuda().eval()
    fr = [f.cuda() for f in O.synth_frames(6, 1, h + pt + pb, w + pl + pr, seed=9, smooth=True)]
    with torch.no_grad():
        outs = net(*fr)
    imgs = [tensor2img_u8(outs[k], crop=(pt, pl, h, w)) for k in (0, 1, 2)]
    files = encode_png(imgs)
    assert encode_png_async(imgs).result() == files
    for img, f in zip(imgs, files):
        _check_file(f, img.cpu().numpy())
    a = imgs[1].cpu().numpy()
    p_np, p_cuda = tmp_path / "np.png", tmp_path / "cuda.png"
    assert imwrite(str(p_np), a) and imwrite(p_cuda, imgs[1])
    assert p_np.read_bytes() == p_cuda.read_bytes() == files[1]
    assert not imwrite(str(tmp_path / "missing_dir" / "x.png"), a)
    try:
        import cv2
    except ImportError:
        return
    from bin_b200.png import install_cv2_imwrite
    original = cv2.imwrite
    try:
        install_cv2_imwrite()
        wrapped = cv2.imwrite
        install_cv2_imwrite()
        assert cv2.imwrite is wrapped and wrapped._bin_b200_original is original
        assert cv2.imwrite(str(tmp_path / "via_cv2.png"), a)
        assert (tmp_path / "via_cv2.png").read_bytes() == files[1]
        assert cv2.imwrite(str(tmp_path / "via_cv2.jpg"), a)
        assert (tmp_path / "via_cv2.jpg").read_bytes()[:2] == b"\xff\xd8"
        assert np.array_equal(cv2.imread(str(tmp_path / "via_cv2.png")), a)
    finally:
        cv2.imwrite = original


def test_refusals():
    from bin_b200 import BinB200Error
    from bin_b200.png import encode_png, imwrite
    good = torch.zeros((8, 9, 3), dtype=torch.uint8, device="cuda")
    bad = [
        [good.cpu()],
        [good.float()],
        [torch.zeros((8, 9, 4), dtype=torch.uint8, device="cuda")],
        [torch.zeros((8, 9), dtype=torch.uint8, device="cuda")],
        [torch.zeros((9, 8, 3), dtype=torch.uint8, device="cuda").transpose(0, 1)],
        [good, torch.zeros((8, 10, 3), dtype=torch.uint8, device="cuda")],
        [],
    ]
    for imgs in bad:
        with pytest.raises(BinB200Error):
            encode_png(imgs)
    with pytest.raises(BinB200Error):
        imwrite("x.jpg", good)
    with pytest.raises(BinB200Error):
        imwrite("x.png", good, [16, 3])
