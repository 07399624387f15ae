"""`simple_knn._C.distCUDA2` (exact 3-nearest-neighbour mean squared distance) without a GPU.

* the CPU oracle (oracle/knn_oracle.c) is bit-identical to a numpy float32 restatement of the contract over all pairs,
  on every test distribution at P <= 3000, and agrees with scipy's cKDTree at 200 000 points;
* the pruning bound of the kernels (gh_knn_math.h, compiled for the host by tests/host_harness/knn_host.cpp) never
  exceeds the float32 distance of a point inside the box, also where dx cancels most of the bits;
* the C ABI: the workspace size needs no GPU, bad arguments are rejected before anything is launched;
* importing the drop-in package loads neither the native library nor CUDA, and never the oracle.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import _knn_cases as K

ROOT = K.ROOT
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import knn_oracle  # noqa: E402

HARNESS_SRC = os.path.join(ROOT, "tests", "host_harness", "knn_host.cpp")
HARNESS_SO = os.path.join(ROOT, "tests", "host_harness", "libknn_host.so")
MATH_H = os.path.join(ROOT, "gaussianhaircut_b200", "csrc", "gh_knn_math.h")


@pytest.fixture(scope="module")
def host():
    newest = max(os.path.getmtime(HARNESS_SRC), os.path.getmtime(MATH_H))
    if not os.path.isfile(HARNESS_SO) or os.path.getmtime(HARNESS_SO) < newest:
        subprocess.run(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-std=c++17", "-w", HARNESS_SRC, "-o",
                        HARNESS_SO], check=True)
    return C.CDLL(HARNESS_SO)


@pytest.fixture(scope="module")
def lib():
    from gaussianhaircut_b200 import build, _capi
    build.build(verbose=False)
    return _capi.load()


# ------------------------------------------------------------------------------------------------------ the oracle
@pytest.mark.parametrize("name", list(K.CASES))
def test_oracle_is_the_contract_bit_for_bit(name):
    gen, n_cpu, _ = K.CASES[name]
    pts = gen(n_cpu, 1)
    K.assert_same_bits(knn_oracle.mean_dist3(pts), K.brute_mean_dist3(pts), name)


@pytest.mark.parametrize("P", range(6))
def test_oracle_small_clouds(P):
    pts = K.tiny(P, 2)
    got = knn_oracle.mean_dist3(pts)
    K.assert_same_bits(got, K.brute_mean_dist3(pts), f"P={P}")
    if P <= 3:
        assert np.all(got == np.inf)           # fewer than three neighbours
    else:
        assert np.all(np.isfinite(got))


def test_oracle_nonfinite_rows_are_nobodys_neighbour():
    pts = np.array([[0, 0, 0], [1, 0, 0], [np.nan, 0, 0], [0, 2, 0], [0, 0, -np.inf], [np.inf, 0, 0], [0, 0, 3]],
                   np.float32)
    got = knn_oracle.mean_dist3(pts)
    assert np.isnan(got[[2, 4, 5]]).all()
    assert got[0] == np.float32((np.float32(1 + 4) + 9) / np.float32(3))
    # the same cloud without the non-finite rows gives the same results for the finite ones
    K.assert_same_bits(got[[0, 1, 3, 6]], knn_oracle.mean_dist3(pts[[0, 1, 3, 6]]))


def _kdtree_contract(pts: np.ndarray, margin: float = 1e-5) -> np.ndarray:
    """The contract, evaluated on the candidates whose float64 squared distance lies within `margin` (relative) of the
    third neighbour's, found by scipy's cKDTree: the three smallest float32 distances are always among them."""
    from scipy.spatial import cKDTree
    fin = np.isfinite(pts).all(axis=1)
    q32 = pts[fin]
    q = q32.astype(np.float64)
    n = q.shape[0]
    tree = cKDTree(q)
    k = 12
    d, nb = tree.query(q, k=k + 1)
    rows = np.arange(n)
    self_mask = nb == rows[:, None]
    d2 = np.where(self_mask, np.inf, d * d)
    d2_sorted = np.sort(d2, axis=1)
    thr = d2_sorted[:, 2] * (1 + margin)
    res = np.empty(n, np.float32)

    def contract(i, cand):
        c = q32[cand]
        dx, dy, dz = c[:, 0] - q32[i, 0], c[:, 1] - q32[i, 1], c[:, 2] - q32[i, 2]
        s = np.sort(np.concatenate([(dx * dx + dy * dy) + dz * dz, np.full(3, np.inf, np.float32)]))[:3]
        return ((s[0] + s[1]) + s[2]) / np.float32(3.0)

    complete = d2_sorted[:, -1] > thr           # the k neighbours returned reach past the margin
    cand = np.where((d2 <= thr[:, None]) & ~self_mask, nb, -1)
    for i in np.nonzero(complete)[0]:
        res[i] = contract(i, cand[i][cand[i] >= 0])
    for i in np.nonzero(~complete)[0]:          # ties or near-ties beyond k: ask for the whole ball
        ball = np.array(tree.query_ball_point(q[i], np.sqrt(thr[i]) * (1 + 1e-12)))
        res[i] = contract(i, ball[ball != i])
    out = np.full(pts.shape[0], np.nan, np.float32)
    out[fin] = res
    return out


@pytest.mark.parametrize("name", ["a_uniform", "b_head_shell", "c_strands"])
def test_oracle_agrees_with_ckdtree_at_200k(name):
    pts = K.CASES[name][0](200_000, 3)
    K.assert_same_bits(knn_oracle.mean_dist3(pts), _kdtree_contract(pts), name)


# ---------------------------------------------------------------------------------------------- the pruning bound
def _boxes(rng, n, centre, extent):
    a = (centre + (rng.random((n, 3)) - 0.5) * extent).astype(np.float32)
    b = (centre + (rng.random((n, 3)) - 0.5) * extent).astype(np.float32)
    lo, hi = np.minimum(a, b), np.maximum(a, b)
    # some degenerate axes (a flat or point-like box)
    flat = rng.random((n, 3)) < 0.1
    hi[flat] = lo[flat]
    return lo, hi


@pytest.mark.parametrize("centre,extent", [((0.0, 0.0, 0.0), 2.0), ((1e4, -1e4, 1e4), 1e-2), ((0.0, 0.0, 0.0), 1e-30),
                                           ((3.0, 0.5, -7.0), 1e3)], ids=["unit", "offset", "underflow", "wide"])
def test_box_bound_never_exceeds_a_distance_inside_the_box(host, centre, extent):
    rng = np.random.default_rng(11)
    n = 200_000
    centre = np.array(centre)
    lo, hi = _boxes(rng, n, centre, extent)
    # queries inside, near and far outside the box
    p = (centre + (rng.random((n, 3)) - 0.5) * extent * rng.choice([0.5, 1.0, 3.0, 100.0], (n, 1))).astype(np.float32)
    bound = np.empty(n, np.float32)
    host.gh_host_knn_box_bound(n, p.ctypes.data, lo.ctypes.data, hi.ctypes.data, bound.ctypes.data)
    worst = np.full(n, np.inf, np.float32)
    for t in range(8):
        # points inside the box: its corners (t < 2) and random interior points, rounded to float32 and clamped
        if t == 0:
            q = lo.copy()
        elif t == 1:
            q = hi.copy()
        else:
            q = (lo + rng.random((n, 3)) * (hi.astype(np.float64) - lo)).astype(np.float32)
            q = np.minimum(np.maximum(q, lo), hi)
        s = np.empty(n, np.float32)
        host.gh_host_knn_dist2(n, p.ctypes.data, q.ctypes.data, s.ctypes.data)
        K.assert_same_bits(s, _dist2_np(p, q), "gh_knn_dist2 vs the contract's s")
        worst = np.minimum(worst, s)
    bad = np.nonzero(bound > worst)[0]
    assert bad.size == 0, f"bound above a distance inside the box: {bound[bad[:4]]} > {worst[bad[:4]]}"
    # the bound is tight where it can be: 0 for a query inside its box
    inside = ((p >= lo) & (p <= hi)).all(axis=1)
    assert inside.any() and np.all(bound[inside] == 0)


def _dist2_np(p, q):
    d = q - p
    return (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]


def test_box_bound_of_the_empty_box_is_infinite(host):
    p = np.zeros((1, 3), np.float32)
    lo = np.full((1, 3), np.inf, np.float32)
    hi = np.full((1, 3), -np.inf, np.float32)
    out = np.empty(1, np.float32)
    host.gh_host_knn_box_bound(1, p.ctypes.data, lo.ctypes.data, hi.ctypes.data, out.ctypes.data)
    assert out[0] == np.inf


# ------------------------------------------------------------------------------------------------------- the C ABI
def test_workspace_size_without_gpu(lib):
    from gaussianhaircut_b200 import _capi
    b = C.c_size_t()
    assert lib.gh_knn_workspace_size(0, C.byref(b)) == 0 and b.value > 0
    sizes = []
    for P in (1, 32, 33, 1_000_000, 4_000_000):
        assert lib.gh_knn_workspace_size(P, C.byref(b)) == 0
        # 16 B per sorted point + a tree of 2 * 2^D boxes of 32 B, 2^D >= P / 32
        leaves = 1 << max(0, int(np.ceil(np.log2(max(1, -(-P // 32))))))
        assert 16 * P + 64 * leaves <= b.value <= 16 * P + 64 * leaves + 1024
        sizes.append(b.value)
    assert sizes == sorted(sizes)
    for P in (-1, 1 << 31):
        assert lib.gh_knn_workspace_size(P, C.byref(b)) == _capi.GH_E_INVALID_ARG
        assert b"P must lie in" in lib.gh_last_error()


def test_entry_points_reject_bad_arguments_before_any_launch(lib):
    from gaussianhaircut_b200 import _capi
    fake, fake8 = C.c_void_p(0x10000), C.c_void_p(0x20000)
    b = C.c_size_t()
    lib.gh_knn_workspace_size(1000, C.byref(b))
    n0 = lib.gh_kernel_launch_count()
    cases = [
        (lib.gh_knn_morton, (-1, fake, fake8, fake, b.value, None), b"P must lie in"),
        (lib.gh_knn_morton, (1000, None, fake8, fake, b.value, None), b"missing points"),
        (lib.gh_knn_morton, (1000, fake, fake8, fake, b.value - 1, None), b"workspace smaller"),
        (lib.gh_knn_morton, (1000, fake, C.c_void_p(0x20004), fake, b.value, None), b"codes must be"),
        (lib.gh_knn_morton, (1000, C.c_void_p(0x10002), fake8, fake, b.value, None), b"4-byte aligned"),
        (lib.gh_knn_mean_dist3, (1000, fake, None, fake, fake, b.value, None), b"order must be"),
        (lib.gh_knn_mean_dist3, (1000, fake, fake8, None, fake, b.value, None), b"out must be"),
        (lib.gh_knn_mean_dist3, (1000, fake, fake8, fake, None, b.value, None), b"missing points or workspace"),
        (lib.gh_knn_mean_dist3, (1 << 31, fake, fake8, fake, fake, b.value, None), b"P must lie in"),
    ]
    for fn, args, msg in cases:
        assert fn(*args) == _capi.GH_E_INVALID_ARG, msg
        assert msg in lib.gh_last_error(), (msg, lib.gh_last_error())
    # P = 0 needs no pointer and launches nothing
    assert lib.gh_knn_morton(0, None, None, None, 0, None) == 0
    assert lib.gh_knn_mean_dist3(0, None, None, None, None, 0, None) == 0
    assert lib.gh_kernel_launch_count() == n0


# ---------------------------------------------------------------------------------------------- the drop-in package
_IMPORT_PROBE = r"""
import sys
sys.path.insert(0, ROOT)
import torch
import gaussianhaircut_b200._capi as capi
capi.LIB_PATH = "/nonexistent/libgh_raster.so"
{prelude}
from simple_knn._C import distCUDA2
from gaussianhaircut_b200.knn import mean_dist3
assert distCUDA2 is mean_dist3
assert capi._lib is None, "importing simple_knn loaded the native library"
assert not torch.cuda.is_initialized(), "importing simple_knn initialised CUDA"
assert "oracle" not in sys.modules and "knn_oracle" not in sys.modules
msgs = []
for x in (torch.zeros(4, 3), torch.zeros(4, 2), torch.zeros(4, 3, dtype=torch.float64), torch.zeros(2, 4, 3),
          torch.zeros(0, 3)):
    try:
        distCUDA2(x)
    except RuntimeError as e:
        msgs.append(str(e))
print("|".join(msgs))
assert capi._lib is None and not torch.cuda.is_initialized()
"""


def _probe(prelude: str = "") -> list:
    code = _IMPORT_PROBE.replace("ROOT", repr(ROOT)).replace("{prelude}", prelude)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=ROOT, timeout=300)
    assert r.returncode == 0, r.stderr[-3000:]
    return r.stdout.strip().split("|")


def test_simple_knn_imports_without_library_or_cuda_and_rejects_bad_input():
    msgs = _probe()
    assert len(msgs) == 5
    assert "no CPU path" in msgs[0] and "no CPU path" in msgs[4]
    assert "shape (P, 3)" in msgs[1] and "shape (P, 3)" in msgs[3]
    assert "Float" in msgs[2]


def test_reference_stub_installer_binds_the_drop_in():
    """oracle/ref_python.install_stubs() stubs only what it cannot find: with this repository on sys.path it now finds
    simple_knn, so the reference's `scene.gaussian_model` binds the real function -- still without side effects."""
    prelude = ("sys.path.insert(0, ROOT + '/oracle'); import ref_python; ref_python.install_stubs(); "
               "import simple_knn; assert simple_knn.__file__.startswith(ROOT)").replace("ROOT", repr(ROOT))
    assert "no CPU path" in _probe(prelude)[0]


def test_drop_in_never_imports_the_oracle():
    files = [os.path.join(ROOT, "simple_knn", f) for f in os.listdir(os.path.join(ROOT, "simple_knn")) if f.endswith(".py")]
    files += [os.path.join(ROOT, "gaussianhaircut_b200", "knn.py"), os.path.join(ROOT, "gaussianhaircut_b200", "csrc", "gh_knn.cu")]
    for f in files:
        src = open(f).read()
        assert "oracle" not in src and "build_ref" not in src, f
