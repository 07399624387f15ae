"""The mesh signed distance (`pysdf.SDF`, `gaussianhaircut_b200.mesh`) without a GPU.

* the float64 oracle (tests/_sdf64.py) is pinned by closed forms: an axis-aligned box, a regular tetrahedron, and the
  vertex, edge and face Voronoi regions of one triangle;
* the kernels' per-face arithmetic (gh_mesh_math.h, compiled for the host by tests/host_harness/sdf_host.cpp): the
  record is the oracle's float32 restatement bit for bit, and every (point, face) distance and solid angle lies within
  the oracle's derived bound;
* the C ABI: the workspace size needs no GPU, bad arguments are refused before anything is launched;
* importing the drop-in package or the module loads neither the native library nor CUDA, and never the oracle.
"""
import ctypes as C
import math
import os
import subprocess
import sys

import numpy as np
import pytest

import _sdf64 as O
import _sdf_cases as K

ROOT = K.ROOT
HARNESS_SRC = os.path.join(ROOT, "tests", "host_harness", "sdf_host.cpp")
HARNESS_SO = os.path.join(ROOT, "tests", "host_harness", "libsdf_host.so")
MATH_H = os.path.join(ROOT, "gaussianhaircut_b200", "csrc", "gh_mesh_math.h")
SMALL = ["icosphere", "head", "head_holes", "degenerate"]


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


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


# ------------------------------------------------------------------------------------------------------ the oracle
def _box():
    h = np.array([0.03, 0.05, 0.02])
    s = np.array([[x, y, z] for x in (-1, 1) for y in (-1, 1) for z in (-1, 1)], np.float64)
    v = (s * h).astype(np.float32)
    h = np.abs(v[7]).astype(np.float64)              # the half extents the float32 box has
    # vertex index = 4 (x > 0) + 2 (y > 0) + (z > 0); faces counter-clockwise seen from outside
    quads = [(0, 1, 3, 2), (4, 6, 7, 5), (0, 4, 5, 1), (2, 3, 7, 6), (0, 2, 6, 4), (1, 5, 7, 3)]
    f = np.array([t for q in quads for t in ((q[0], q[1], q[2]), (q[0], q[2], q[3]))], np.int32)
    return v, f, h


def test_oracle_box_closed_form():
    v, f, h = _box()
    rng = np.random.default_rng(1)
    p = (rng.uniform(-3, 3, (3000, 3)) * h).astype(np.float32)
    q = np.abs(p.astype(np.float64)) - h
    box_sdf = np.linalg.norm(np.maximum(q, 0), axis=1) + np.minimum(q.max(1), 0)      # negative inside
    o = O.query64(p, v, f)
    np.testing.assert_allclose(o["sdf"], -box_sdf, rtol=0, atol=1e-14)
    inside = box_sdf < 0
    np.testing.assert_allclose(o["w"][inside], 1.0, atol=1e-12)
    np.testing.assert_allclose(o["w"][~inside], 0.0, atol=1e-12)


def test_oracle_regular_tetrahedron():
    v = np.array([[1, 1, 1], [1, -1, -1], [-1, 1, -1], [-1, -1, 1]], np.float32) * np.float32(0.05)
    f = np.array([[0, 1, 2], [0, 3, 1], [0, 2, 3], [1, 3, 2]], np.int32)
    v64 = v.astype(np.float64)
    rng = np.random.default_rng(2)
    bary = rng.dirichlet([1, 1, 1, 1], 500)
    p = (bary @ v64).astype(np.float32)                  # inside: d = the smallest distance to the four face planes
    planes = []
    for a, b, c in f:
        n = np.cross(v64[b] - v64[a], v64[c] - v64[a])
        planes.append((n / np.linalg.norm(n), v64[a]))
    d_in = np.min([np.abs((p - a) @ n) for n, a in planes], axis=0)
    o = O.query64(p, v, f)
    np.testing.assert_allclose(o["sdf"], d_in, rtol=1e-12, atol=1e-16)
    np.testing.assert_allclose(o["w"], 1.0, atol=1e-12)
    # outside, straight above each face's centroid: the distance is the height, the winding number 0
    cen = v64[f].mean(1)
    nrm = np.array([n for n, _ in planes])
    h = rng.uniform(1e-3, 0.1, (4, 1))
    p = (cen + nrm * h).astype(np.float32)
    o = O.query64(p, v, f)
    exact = np.abs(np.einsum("ij,ij->i", p.astype(np.float64) - cen, nrm))
    np.testing.assert_allclose(o["sdf"], -exact, rtol=1e-9)
    np.testing.assert_allclose(o["w"], 0.0, atol=1e-12)


def test_oracle_voronoi_regions_of_one_triangle():
    v = np.array([[0, 0, 0], [0.04, 0, 0], [0, 0.03, 0]], np.float32)
    m = O.Mesh64(v, np.array([[0, 1, 2]]))
    p = np.array([[0.01, 0.01, 0.02],            # face region: the height
                  [0.02, -0.01, 0.005],          # edge ab: the distance to the x axis
                  [-0.01, 0.01, -0.003],         # edge ca: the distance to the y axis
                  [-0.01, -0.02, 0.004],         # vertex a
                  [0.06, -0.01, 0.0],            # vertex b
                  [-0.002, 0.05, 0.01],          # vertex c
                  [0.03, 0.03, 0.0]])            # edge bc, in the plane
    bc_dir = np.array([-0.04, 0.03, 0]) / 0.05
    rel = p[6] - np.array([0.04, 0, 0])
    exact = [0.02, math.hypot(0.01, 0.005), math.hypot(0.01, 0.003), math.sqrt(1e-4 + 4e-4 + 1.6e-5),
             math.hypot(0.02, 0.01), math.sqrt(0.002 ** 2 + 0.02 ** 2 + 1e-4),
             np.linalg.norm(rel - (rel @ bc_dir) * bc_dir)]
    got = O.pairs(p.astype(np.float32), m, np.zeros(len(p), int))["d"]
    np.testing.assert_allclose(got, exact, rtol=1e-6)     # p rounded to float32


# ---------------------------------------------------------------------------------------------- the host harness
@pytest.mark.parametrize("name", SMALL + ["big"])
def test_record_is_the_oracles_float32_restatement(host, name):
    v, f = K.MESHES[name]()
    tri = np.ascontiguousarray(v[f].reshape(-1, 9))
    rec = np.empty((len(f), 28), np.float32)
    host.gh_host_sdf_record(len(f), _ptr(tri), _ptr(rec))
    assert np.array_equal(rec.view(np.uint32), O.record32(v, f).view(np.uint32))


def _per_face_points(v, f, rng, n):
    """(points, face): points built on their own face -- on it, above it, beside its edges and vertices."""
    face = rng.integers(0, len(f), n)
    tri = v[f[face]].astype(np.float64)
    nrm = np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0])
    with np.errstate(invalid="ignore", divide="ignore"):
        nrm = np.nan_to_num(nrm / np.linalg.norm(nrm, axis=1, keepdims=True))
    bary = rng.normal(0.33, 0.6, (n, 3))
    bary /= bary.sum(1, keepdims=True)
    scale = 10.0 ** rng.uniform(-8, -1, (n, 1))
    p = np.einsum("nk,nkj->nj", bary, tri) + nrm * rng.normal(0, 1, (n, 1)) * scale \
        + rng.normal(0, 1, (n, 3)) * scale * (rng.random((n, 1)) < 0.3)
    return p.astype(np.float32), face


@pytest.mark.parametrize("name", SMALL)
def test_host_pairs_within_the_derived_bound(host, name):
    v, f = K.MESHES[name]()
    rng = np.random.default_rng(7)
    p1, f1 = _per_face_points(v, f, rng, 60_000)
    q = K.queries(v, f, 2000, 8)
    q = q[np.isfinite(q).all(1)]
    p2 = np.repeat(q, 20, 0)
    f2 = rng.integers(0, len(f), len(p2))
    p, face = np.concatenate([p1, p2]), np.concatenate([f1, f2])
    rec = np.ascontiguousarray(O.record32(v, f)[face])
    d2 = np.empty(len(p), np.float32)
    om = np.empty(len(p), np.float32)
    host.gh_host_sdf_pair(len(p), _ptr(np.ascontiguousarray(p)), _ptr(rec), _ptr(d2), _ptr(om))
    o = O.pairs(p, O.Mesh64(v, f), face)
    err_d = np.abs(np.sqrt(d2.astype(np.float64)) - o["d"])
    err_w = np.abs(om.astype(np.float64) - o["omega"])
    checked = np.isfinite(o["e"])
    assert checked.mean() > 0.99
    r_d, r_w = err_d[checked] / np.maximum(o["e"][checked], 1e-300), err_w / o["domega"]
    print(f"{name}: {len(p)} pairs, largest error / bound: distance {r_d.max():.3g}, solid angle {r_w.max():.3g}")
    assert r_d.max() <= 1.0 and r_w.max() <= 1.0


# ------------------------------------------------------------------------------------------------------- the C ABI
def test_workspace_size_without_gpu(lib):
    from gaussianhaircut_b200 import _capi
    b = C.c_size_t()
    for F in (1, 12, 10_080, (1 << 31) - 1):
        assert lib.gh_sdf_workspace_size(F, C.byref(b)) == 0 and b.value == 112 * F
    for F in (0, -1, 1 << 31):
        assert lib.gh_sdf_workspace_size(F, C.byref(b)) == _capi.GH_E_INVALID_ARG
        assert b"F must lie in [1, 2^31)" in lib.gh_last_error()
    assert lib.gh_sdf_workspace_size(5, None) == _capi.GH_E_INVALID_ARG


def test_entry_points_refuse_bad_arguments_before_any_launch(lib):
    from gaussianhaircut_b200 import _capi
    fv, ff, fs, ws, out = (C.c_void_p(x) for x in (0x10000, 0x20000, 0x30000, 0x40000, 0x50000))
    F = 100
    nb = 112 * F
    n0 = lib.gh_kernel_launch_count()
    prep, query = lib.gh_sdf_prepare, lib.gh_sdf_query
    cases = [
        (prep, (0, F, fv, ff, ws, nb, fs, 0, None), b"V must lie in"),
        (prep, (1 << 31, F, fv, ff, ws, nb, fs, 0, None), b"V must lie in"),
        (prep, (10, 0, fv, ff, ws, nb, fs, 0, None), b"F must lie in"),
        (prep, (10, 1 << 31, fv, ff, ws, nb, fs, 0, None), b"F must lie in"),
        (prep, (10, F, None, ff, ws, nb, fs, 0, None), b"missing verts"),
        (prep, (10, F, fv, ff, ws, nb, None, 0, None), b"missing verts"),
        (prep, (10, F, C.c_void_p(0x10002), ff, ws, nb, fs, 0, None), b"4-byte aligned"),
        (prep, (10, F, fv, ff, None, nb, fs, 0, None), b"missing workspace"),
        (prep, (10, F, fv, ff, C.c_void_p(0x40008), nb, fs, 0, None), b"16-byte aligned"),
        (prep, (10, F, fv, ff, ws, nb - 1, fs, 0, None), b"workspace of"),
        (query, (-1, fv, F, ws, nb, out, None, None, 0, None), b"N must lie in"),
        (query, (1 << 31, fv, F, ws, nb, out, None, None, 0, None), b"N must lie in"),
        (query, (10, fv, 0, ws, nb, out, None, None, 0, None), b"F must lie in"),
        (query, (10, None, F, ws, nb, out, None, None, 0, None), b"missing points or sdf"),
        (query, (10, fv, F, ws, nb, None, None, None, 0, None), b"missing points or sdf"),
        (query, (10, fv, F, ws, nb, out, C.c_void_p(0x60001), None, 0, None), b"4-byte aligned"),
        (query, (10, fv, F, ws, nb - 112, out, None, None, 0, None), b"workspace of"),
        (query, (10, fv, F, C.c_void_p(0x40004), nb, out, None, None, 0, None), b"16-byte aligned"),
    ]
    for fn, args, msg in cases:
        assert fn(*args) == _capi.GH_E_INVALID_ARG, msg
        assert msg in lib.gh_last_error(), (msg, lib.gh_last_error())
    lib.gh_stage_timing_enable(1)
    try:
        assert query(10, fv, F, ws, nb, out, None, None, 1, None) == _capi.GH_E_INVALID_ARG
        assert b"stage timer" in lib.gh_last_error()
        assert prep(10, F, fv, ff, ws, nb, fs, 1, None) == _capi.GH_E_INVALID_ARG
    finally:
        lib.gh_stage_timing_enable(0)
    assert query(0, None, F, ws, nb, None, None, None, 0, None) == 0      # N = 0 launches nothing
    assert lib.gh_kernel_launch_count() == n0


# ---------------------------------------------------------------------------------------------- the drop-in package
_IMPORT_PROBE = r"""
import sys
sys.path.insert(0, ROOT)
import torch
import gaussianhaircut_b200._capi as capi
capi.LIB_PATH = "/nonexistent/libgh_raster.so"
import pysdf
from pysdf import SDF
from gaussianhaircut_b200 import mesh
assert SDF is pysdf.SDF and pysdf.MeshSDF is mesh.MeshSDF
assert capi._lib is None, "importing pysdf loaded the native library"
assert not torch.cuda.is_initialized(), "importing pysdf initialised CUDA"
assert not any(k in sys.modules for k in ("oracle", "_sdf64", "_sdf_cases"))
msgs = []
for v, f in (([[0, 0, 0]] * 3, [[0, 1]]), ([[0, 0, 0]] * 3, [[0.0, 1.0, 2.0]]), ([[0, 0, 0]] * 3, [[0, 1, 3]]),
             ([[0, 0, 0], [1, 0, 0], [0, 1, 0]], [[0, 1, 2]])):
    try:
        SDF(v, f)
    except RuntimeError as e:
        msgs.append(type(e).__name__ + ": " + str(e))
print("|".join(msgs))
"""


def test_pysdf_imports_without_library_or_cuda_and_refuses_bad_input():
    code = _IMPORT_PROBE.replace("ROOT", repr(ROOT))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=ROOT, timeout=300)
    assert r.returncode == 0, r.stderr[-3000:]
    msgs = r.stdout.strip().split("|")
    assert len(msgs) == 4
    assert "(F, 3)" in msgs[0] and "integer" in msgs[1] and "outside [0, 3)" in msgs[2]
    assert msgs[3].startswith("RuntimeError")        # no CUDA, or no library: never a CPU answer


def test_product_never_imports_the_oracle():
    files = [os.path.join(ROOT, "pysdf", "__init__.py"), os.path.join(ROOT, "gaussianhaircut_b200", "mesh.py"),
             os.path.join(ROOT, "gaussianhaircut_b200", "csrc", "gh_sdf.cu")]
    for f in files:
        src = open(f).read()
        assert "oracle" not in src and "_sdf64" not in src and "_sdf_cases" not in src, f
