"""Hair orientation maps (`gaussianhaircut_b200.orient`) without a GPU.

* the bank: the oracle's restatement of scikit-image's Gabor kernel matches OpenCV's independent one per angle, with and
  without a phase offset; the product's `gabor_bank` is bit-identical to the oracle's; K = 17 and the per-angle supports
  at the defaults are pinned;
* the DoG weights are scipy's own;
* the per-pixel epilogue (gh_orient_math.h, compiled for the host by tests/host_harness/orient_host.cpp) agrees bit for
  bit with a numpy float32 restatement of the reference's torch expressions, at ties, zeros, wrap-around and G > 1;
* the C ABI rejects bad arguments before anything is launched;
* importing the module loads neither the native library nor CUDA, and never the oracle.
"""
import ctypes as C
import math
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import orient64  # noqa: E402

from gaussianhaircut_b200 import orient  # noqa: E402

HARNESS_SRC = os.path.join(ROOT, "tests", "host_harness", "orient_host.cpp")
HARNESS_SO = os.path.join(ROOT, "tests", "host_harness", "liborient_host.so")
MATH_H = os.path.join(ROOT, "gaussianhaircut_b200", "csrc", "gh_orient_math.h")


@pytest.fixture(scope="module")
def host():
    newest = max(os.path.getmtime(HARNESS_SRC), os.path.getmtime(MATH_H))
    if not os.path.isfile(HARNESS_SO) or os.path.getmtime(HARNESS_SO) < newest:
        subprocess.run(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-std=c++17", "-w", HARNESS_SRC, "-o",
                        HARNESS_SO], check=True)
    h = C.CDLL(HARNESS_SO)
    h.gh_host_orient_epilogue.argtypes = [C.c_int, C.c_int, C.c_int] + [C.c_void_p] * 4
    h.gh_host_orient_epilogue.restype = None
    return h


@pytest.fixture(scope="module")
def lib():
    from gaussianhaircut_b200 import build, _capi
    build.build(verbose=False)
    return _capi.load()


# ------------------------------------------------------------------------------------------------------------ bank
def _cv2_gabor(f, theta, sx, sy, offset, shape):
    """OpenCV's real Gabor kernel in scikit-image's normalisation.  OpenCV stores the value at (x, y) in element
    (ymax - y, xmax - x), i.e. rotated by 180 degrees against scikit-image; an even kernel (offset 0) does not see it."""
    cv2 = pytest.importorskip("cv2")
    h, w = shape
    k = cv2.getGaborKernel((w, h), sx, theta, 1.0 / f, sx / sy, offset, cv2.CV_64F) / (2 * math.pi * sx * sy)
    return k[::-1, ::-1]


@pytest.mark.parametrize("offset", [0.0, math.pi / 2, 1.0])
@pytest.mark.parametrize("sx,sy,f", [(1.8, 2.4, 0.23), (1.0, 2.4, 0.5), (2.0, 1.0, 1.0)])
def test_oracle_gabor_kernel_matches_opencv(offset, sx, sy, f):
    worst = 0.0
    for t in np.linspace(0, math.pi * 179 / 180, 180):
        k = np.real(orient64.gabor_kernel(f, theta=math.pi - t, sigma_x=sx, sigma_y=sy, offset=offset))
        worst = max(worst, float(np.abs(k - _cv2_gabor(f, math.pi - t, sx, sy, offset, k.shape)).max()))
    assert worst <= 1e-15, worst


@pytest.mark.parametrize("kw", [{}, {"num_sigmas_x": 2, "num_offsets": 2}, {"num_frequencies": 2},
                                {"num_sigmas_y": 2, "num_filters": 90}, {"num_filters": 256}])
def test_product_bank_is_the_oracle_bank_bit_for_bit(kw):
    bank, thetas = orient.gabor_bank(**kw)
    ob, ot, G = orient64.bank(**kw)
    assert bank.dtype == np.float32 and thetas.dtype == np.float32
    assert bank.shape == ob.shape and bank.shape[0] == G * len(thetas)
    assert np.array_equal(bank.view(np.uint32), ob.view(np.uint32))
    assert np.array_equal(thetas.view(np.uint32), ot.view(np.uint32))


# (first theta index, last, x0, y0) at the defaults (sigma_x 1.8, sigma_y 2.4): kernel j spans (2*y0+1) x (2*x0+1)
DEFAULT_SUPPORTS = [(0, 13, 6, 8), (14, 22, 6, 7), (23, 33, 5, 7), (34, 43, 5, 6), (44, 46, 6, 6), (47, 56, 6, 5),
                    (57, 67, 7, 5), (68, 76, 7, 6), (77, 103, 8, 6), (104, 112, 7, 6), (113, 123, 7, 5),
                    (124, 133, 6, 5), (134, 136, 6, 6), (137, 146, 5, 6), (147, 157, 5, 7), (158, 166, 6, 7),
                    (167, 179, 6, 8)]


def test_default_bank_shape_and_supports():
    bank, thetas = orient.gabor_bank()
    assert bank.shape == (180, 17, 17) and thetas.shape == (180,)
    taps = 0
    for a, b, x0, y0 in DEFAULT_SUPPORTS:
        for j in range(a, b + 1):
            assert orient64.support(1.8, 2.4, math.pi - float(np.float64(j) * math.pi / 180)) == (x0, y0), j
            k = orient64.gabor_kernel(0.23, theta=math.pi - np.linspace(0, math.pi * 179 / 180, 180)[j], sigma_x=1.8,
                                      sigma_y=2.4)
            assert k.shape == (2 * y0 + 1, 2 * x0 + 1)
            # the padded filter is zero outside its centred support
            ys, xs = np.nonzero(bank[j])
            assert ys.min() >= 8 - y0 and ys.max() <= 8 + y0 and xs.min() >= 8 - x0 and xs.max() <= 8 + x0
            taps += (2 * x0 + 1) * (2 * y0 + 1)
    assert taps == 32948                            # of 180 * 289 = 52020 dense


def test_dog_weights_are_scipys():
    from scipy.ndimage import _filters
    for s in (0.4, 1.0, 2.5, 10.0, 13.3):
        r = int(4.0 * s + 0.5)
        assert np.array_equal(orient.gaussian_weights(s), _filters._gaussian_kernel1d(s, 0, r))


# -------------------------------------------------------------------------------------------------------- epilogue
def _epilogue_np(F: np.ndarray, thetas: np.ndarray, nf: int, G: int):
    """The reference's torch expressions (calc_orientation_maps.py:79-90) restated in numpy float32, both sums in
    increasing j: F (n, nf*G) in channel order j*G + g -> (idx int64, var float32)."""
    n = F.shape[0]
    Fg = F.reshape(n, nf, G)
    pi = np.float32(math.pi)
    best_i = np.zeros(n, np.int64)
    best_v = np.zeros(n, np.float32)
    for g in range(G):
        f = Fg[:, :, g]
        idx = f.argmax(axis=1)
        a = (idx.astype(np.float32) / np.float32(nf)) * pi
        S = np.zeros(n, np.float32)
        for j in range(nf):
            S = S + f[:, j]
        S = np.maximum(S, np.float32(1e-12))
        var = np.zeros(n, np.float32)
        for j in range(nf):
            t = a - thetas[j]
            d = np.minimum(np.abs(t), np.minimum(np.abs(t - pi), np.abs(t + pi)))
            var = var + (d * d) * (f[:, j] / S)
        take = (var < best_v) | (g == 0)
        best_i = np.where(take, idx, best_i)
        best_v = np.where(take, var, best_v)
    return best_i, best_v


def _host_epilogue(host, F, thetas, nf, G):
    F = np.ascontiguousarray(F, np.float32)
    idx = np.empty(F.shape[0], np.int64)
    var = np.empty(F.shape[0], np.float32)
    host.gh_host_orient_epilogue(F.shape[0], nf, G, F.ctypes.data, thetas.ctypes.data, idx.ctypes.data, var.ctypes.data)
    return idx, var


def _cases(nf, G, rng):
    n = 4000
    F = np.abs(rng.standard_normal((n, nf * G)).astype(np.float32)) * rng.choice([1e-3, 1.0, 1e3], (n, 1)).astype(np.float32)
    F[0] = 0                                            # all-zero responses: index 0, variance 0
    F[1] = 1.0                                          # all tied: first index
    F[2, :] = 0.5
    F[2, 5 * G::7 * G] = 2.0                            # ties at the maximum: the first of them
    F[3] = 0.1
    F[3, 0] = 3.0                                       # argmax at 0: distances wrap at pi
    F[4] = 0.1
    F[4, (nf - 1) * G] = 3.0                            # argmax at nf - 1
    F[5] = rng.random(nf * G).astype(np.float32) * np.float32(1e-30)   # tiny sums: the 1e-12 clamp
    if G > 1:
        F[6:200] = np.tile(F[6:200, :G * nf].reshape(-1, nf, G)[:, :, :1], (1, 1, G)).reshape(-1, nf * G)  # tied groups
        F[200:300, 1::G] = F[200:300, 0::G][:, ::-1]    # mirrored responses: equal variance, different index
    return F


@pytest.mark.parametrize("nf,G", [(180, 1), (180, 4), (7, 3), (1, 2), (256, 1)])
def test_epilogue_matches_the_reference_expressions_bit_for_bit(host, nf, G):
    rng = np.random.default_rng(nf * 10 + G)
    thetas = np.linspace(0, math.pi * (nf - 1) / nf, nf).astype(np.float32)
    F = _cases(nf, G, rng)
    idx, var = _host_epilogue(host, F, thetas, nf, G)
    want_i, want_v = _epilogue_np(F, thetas, nf, G)
    assert np.array_equal(idx, want_i)
    assert np.array_equal(var.view(np.uint32), want_v.view(np.uint32))
    assert idx[0] == 0 and var[0] == 0 and idx[1] == 0
    if nf > 7 and G == 1:
        assert idx[2] == 5 and idx[3] == 0 and idx[4] == nf - 1
    if G > 1:
        assert np.all(idx[6:200] == want_i[6:200])


def test_epilogue_distance_wraps_at_pi(host):
    nf = 180
    thetas = np.linspace(0, math.pi * 179 / 180, 180).astype(np.float32)
    F = np.zeros((2, nf), np.float32)
    F[0, 0] = 1.0
    F[0, 179] = 0.5                                     # one degree away across the wrap
    F[1, 179] = 1.0
    F[1, 0] = 0.5
    idx, var = _host_epilogue(host, F, thetas, nf, 1)
    assert list(idx) == [0, 179]
    one_deg = np.float32(math.pi) / 180
    assert np.allclose(var, (one_deg ** 2) * 0.5 / 1.5, rtol=1e-5)


# ------------------------------------------------------------------------------------------------------- the C ABI
def test_workspace_size_without_gpu(lib):
    from gaussianhaircut_b200 import _capi
    b = C.c_size_t()
    assert lib.gh_orient_workspace_size(1080, 1920, 180, 17, 180, C.byref(b)) == 0
    npix = 1080 * 1920
    assert b.value >= npix * (4 + 3 * 8) + 3 * 64 * 289 * 4
    for args in ((0, 5, 180, 17, 180), (5, -1, 180, 17, 180), (1 << 16, 1 << 15, 180, 17, 180), (5, 5, 180, 16, 180),
                 (5, 5, 180, 19, 180), (5, 5, 180, 17, 257), (5, 5, 181, 17, 180), (5, 5, 4096 + 256, 17, 256)):
        assert lib.gh_orient_workspace_size(*args, C.byref(b)) == _capi.GH_E_INVALID_ARG, args


def test_entry_points_reject_bad_arguments_before_any_launch(lib):
    from gaussianhaircut_b200 import _capi
    H, W = 64, 48
    b = C.c_size_t()
    assert lib.gh_orient_workspace_size(H, W, 720, 17, 180, C.byref(b)) == 0
    n = b.value
    b0 = C.c_size_t()
    lib.gh_orient_workspace_size(H, W, 0 + 180, 17, 180, C.byref(b0))
    img, wl, wh, dog = C.c_void_p(0x10000), C.c_void_p(0x20000), C.c_void_p(0x30000), C.c_void_p(0x40000)
    ws, bank, th, o, v = C.c_void_p(0x100000), C.c_void_p(0x50000), C.c_void_p(0x60000), C.c_void_p(0x70000), C.c_void_p(0x80000)
    dog_ok = (H, W, 3, img, wl, 2, wh, 40, dog, ws, n, None)
    gab_ok = (H, W, bank, 720, 17, 180, th, o, v, ws, n, None)

    def dog_(**kw):
        names = ("H", "W", "C", "img", "wl", "rl", "wh", "rh", "dog", "ws", "n", "s")
        a = dict(zip(names, dog_ok), **kw)
        return lib.gh_orient_dog(*[a[k] for k in names])

    def gab(**kw):
        names = ("H", "W", "bank", "N", "K", "nf", "th", "o", "v", "ws", "n", "s")
        a = dict(zip(names, gab_ok), **kw)
        return lib.gh_orient_gabor(*[a[k] for k in names])

    n0 = lib.gh_kernel_launch_count()
    cases = [
        (dog_, dict(H=0), b"H and W must be positive"), (dog_, dict(W=-3), b"H and W must be positive"),
        (dog_, dict(H=1 << 16, W=1 << 15), b"H*W < 2^31"), (dog_, dict(C=1), b"C must be 3"),
        (dog_, dict(C=2), b"C must be 3"), (dog_, dict(rl=-1), b"radii"), (dog_, dict(rh=5000), b"radii"),
        (dog_, dict(img=None), b"missing image"), (dog_, dict(wl=None), b"missing image"),
        (dog_, dict(dog=None), b"missing image"), (dog_, dict(dog=C.c_void_p(0x40004)), b"8-byte aligned"),
        (dog_, dict(wh=C.c_void_p(0x30004)), b"8-byte aligned"), (dog_, dict(ws=None), b"256-byte aligned"),
        (dog_, dict(ws=C.c_void_p(0x100010)), b"256-byte aligned"), (dog_, dict(n=100), b"workspace smaller"),
        (gab, dict(H=-1), b"H and W must be positive"), (gab, dict(K=16), b"K must be odd"),
        (gab, dict(K=19), b"K must be odd"), (gab, dict(K=0), b"K must be odd"), (gab, dict(nf=257, N=257), b"num_filters"),
        (gab, dict(N=721), b"num_filters"), (gab, dict(N=4096 + 256, nf=256), b"num_filters"),
        (gab, dict(nf=0), b"num_filters"), (gab, dict(bank=None), b"missing bank"), (gab, dict(th=None), b"missing bank"),
        (gab, dict(o=None), b"missing bank"), (gab, dict(v=None), b"missing bank"),
        (gab, dict(o=C.c_void_p(0x70004)), b"8-byte aligned"), (gab, dict(bank=C.c_void_p(0x50002)), b"4-byte aligned"),
        (gab, dict(ws=C.c_void_p(0x100080)), b"256-byte aligned"), (gab, dict(n=n - 1), b"workspace smaller"),
        (gab, dict(n=b0.value), b"workspace smaller"),
    ]
    for fn, kw, msg in cases:
        assert fn(**kw) == _capi.GH_E_INVALID_ARG, (kw, msg)
        assert msg in lib.gh_last_error(), (kw, msg, lib.gh_last_error())
    assert lib.gh_kernel_launch_count() == n0


# ---------------------------------------------------------------------------------------------- the drop-in module
_IMPORT_PROBE = r"""
import sys
sys.path.insert(0, ROOT)
import numpy as np
import torch
import gaussianhaircut_b200._capi as capi
capi.LIB_PATH = "/nonexistent/libgh_raster.so"
from gaussianhaircut_b200 import orient
from gaussianhaircut_b200.orient import orientation_maps, calc_orients, gabor_bank
assert capi._lib is None, "importing orient loaded the native library"
assert not torch.cuda.is_initialized(), "importing orient initialised CUDA"
assert "orient64" not in sys.modules and "oracle" not in sys.modules
bank, thetas = gabor_bank()
msgs = []
for x in (torch.zeros(4, 4, 3, dtype=torch.uint8), torch.zeros(4, 4, 2, dtype=torch.uint8), torch.zeros(4, 4, 3),
          torch.zeros(4, 4, dtype=torch.uint8), np.zeros((4, 4, 3), np.uint8)):
    try:
        orientation_maps(x)
    except RuntimeError as e:
        msgs.append(str(e))
try:
    calc_orients(np.zeros((4, 4, 3), np.float32), 0.4, 10, 1, 180, 1, 1, 1, 64)
except RuntimeError as e:
    msgs.append(str(e))
print("|".join(msgs))
assert capi._lib is None and not torch.cuda.is_initialized()
"""


def test_orient_imports_without_library_or_cuda_and_rejects_bad_input():
    code = _IMPORT_PROBE.replace("ROOT", repr(ROOT))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=ROOT, timeout=300)
    assert r.returncode == 0, r.stderr[-3000:]
    msgs = r.stdout.strip().split("|")
    assert len(msgs) == 6
    assert "no CPU path" in msgs[0]
    assert "shape (H, W, 3)" in msgs[1] and "shape (H, W, 3)" in msgs[3]
    assert "Byte" in msgs[2]
    assert "torch.Tensor" in msgs[4]
    assert "uint8" in msgs[5]


def test_product_never_imports_the_oracle():
    for f in (os.path.join(ROOT, "gaussianhaircut_b200", "orient.py"),
              os.path.join(ROOT, "gaussianhaircut_b200", "csrc", "gh_orient.cu"), MATH_H):
        src = open(f).read()
        assert "oracle" not in src and "orient64" not in src and "build_ref" not in src, f


def test_cli_accepts_the_reference_arguments():
    args = orient.parser().parse_known_args(
        ["--img_path", "a", "--mask_path", "b", "--orient_dir", "c", "--conf_dir", "d", "--filtered_img_dir", "e",
         "--vis_img_dir", "f", "--dog_low", "0.5", "--dog_high", "8", "--num_frequencies", "2", "--num_filters", "90",
         "--num_sigmas_x", "2", "--num_sigmas_y", "1", "--num_offsets", "2", "--patch_size", "32", "--crop_size", "-1",
         "--unknown_flag", "x"])[0]
    assert (args.img_path, args.dog_low, args.dog_high, args.num_filters, args.num_offsets, args.patch_size) == \
        ("a", 0.5, 8.0, 90, 2, 32)
