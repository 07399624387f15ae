"""The mesh rasterizer (csrc/gh_mesh_raster.cu, `gaussianhaircut_b200.mesh`) without a GPU.

* the float64 oracle (tests/_meshraster64.py) is pinned by closed forms: lattice counts of an axis-aligned right
  triangle and of a quad split on its diagonal (centres on an edge are not covered), two coplanar faces, a unit cube,
  faces behind the camera and across its z = 0 plane;
* the kernels' arithmetic (gh_mesh_math.h, compiled for the host by tests/host_harness/mesh_raster_host.cpp): every
  edge function and depth within the oracle's derived bound, coverage equal to the oracle's wherever it is decided, and
  the brute-force z-buffer equal to the oracle at decided pixels and admissible elsewhere, on the test meshes under
  random cameras;
* the numpy restatement of the script's visibility logic on hand cases, and `head_masks` against cv2;
* the C ABI: the workspace size needs no GPU, bad arguments are refused before anything is launched.
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

import _meshraster64 as O
import _sdf_cases as K

ROOT = K.ROOT
HARNESS_SRC = os.path.join(ROOT, "tests", "host_harness", "mesh_raster_host.cpp")
HARNESS_SO = os.path.join(ROOT, "tests", "host_harness", "libmesh_raster_host.so")
MATH_H = os.path.join(ROOT, "gaussianhaircut_b200", "csrc", "gh_mesh_math.h")


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


def _c(a, dt):
    return np.ascontiguousarray(a, dtype=dt)


def brute(host, v, f, Ks, Rs, ts, H, W):
    """-> pix_to_face (B,H,W) int32 and the status bits, from the host harness."""
    Ks, Rs, ts = _c(Ks, np.float32).reshape(-1, 3, 3), _c(Rs, np.float32).reshape(-1, 3, 3), _c(ts, np.float32).reshape(-1, 3)
    out = np.empty((len(Ks), H, W), np.int32)
    st = C.c_uint(0)
    host.gh_host_raster_brute(len(v), len(f), _ptr(_c(v, np.float32)), _ptr(_c(f, np.int32)), len(Ks), _ptr(Ks),
                              _ptr(Rs), _ptr(ts), H, W, _ptr(out), C.byref(st))
    return out, st.value


def pairs(host, v, f, Km, Rm, tm, H, W, face, row, col):
    """Harness setup of one view and evaluation of the given pairs -> code (F,), w (n,3), covered (n,), z (n,)."""
    F = len(f)
    rec = np.zeros((F, 20), np.float32)
    code = np.empty(F, np.int32)
    host.gh_host_raster_setup(len(v), F, _ptr(_c(v, np.float32)), _ptr(_c(f, np.int32)), _ptr(_c(Km, np.float32)),
                              _ptr(_c(Rm, np.float32)), _ptr(_c(tm, np.float32)), H, W, _ptr(rec), _ptr(code))
    n = len(face)
    w = np.empty((n, 3), np.float32)
    cov = np.empty(n, np.int32)
    z = np.empty(n, np.float32)
    host.gh_host_raster_pairs(n, _ptr(rec), _ptr(_c(face, np.int32)), _ptr(_c(row, np.int32)), _ptr(_c(col, np.int32)),
                              _ptr(w), _ptr(cov), _ptr(z))
    return code, w, cov.astype(bool), z


# A camera whose screen coordinates are the world x, y of points at z = 1: every setup operation is exact there.
K1, R1, T1 = np.eye(3, dtype=np.float32), np.eye(3, dtype=np.float32), np.zeros(3, np.float32)


def _screen_mesh(tris):
    v = np.array([[x, y, 1.0] for tri in tris for x, y in tri], np.float32)
    f = np.arange(len(v), dtype=np.int32).reshape(-1, 3)
    return v, f


# ------------------------------------------------------------------------------------------------------ the oracle
def test_oracle_right_triangle_lattice_count(host):
    v, f = _screen_mesh([[(0, 0), (8, 0), (0, 8)]])
    H = W = 12
    o = O.raster64(v, f, K1, R1, T1, H, W)
    i, j = np.mgrid[0:H, 0:W]
    inside = i + j < 7                                  # (j + .5) + (i + .5) < 8
    on_edge = i + j == 7                                # centres on the hypotenuse
    ans = o["answer"].numpy()
    dec = o["decided"].numpy()
    assert inside.sum() == 28 and on_edge.sum() == 8
    assert dec[inside].all() and (ans[inside] == 0).all()
    assert dec[~inside & ~on_edge].all() and (ans[~inside & ~on_edge] == -1).all()
    edge_pairs = on_edge[o["row"].numpy(), o["col"].numpy()]
    assert (o["W"].numpy()[edge_pairs].min(1) == 0).all()   # exactly on the edge: undecided, never certain
    assert not dec[on_edge].any()
    p2f, st = brute(host, v, f, K1, R1, T1, H, W)
    assert st == 0 and np.array_equal(p2f[0] == 0, inside)     # the float32 rule drops the centres on the edge


def test_oracle_quad_diagonal_drops_its_centres(host):
    v, f = _screen_mesh([[(0, 0), (8, 0), (8, 8)], [(0, 0), (8, 8), (0, 8)]])
    H = W = 10
    o = O.raster64(v, f, K1, R1, T1, H, W)
    i, j = np.mgrid[0:H, 0:W]
    sq = (i < 8) & (j < 8)
    lower, upper, diag = sq & (i < j), sq & (i > j), sq & (i == j)
    ans, dec = o["answer"].numpy(), o["decided"].numpy()
    assert dec[lower | upper].all() and (ans[lower] == 0).all() and (ans[upper] == 1).all()
    assert (ans[~sq] == -1).all() and dec[~sq].all()
    p2f, _ = brute(host, v, f, K1, R1, T1, H, W)
    assert np.array_equal(p2f[0], np.where(lower, 0, np.where(upper, 1, -1)))
    assert (p2f[0][diag] == -1).all() and diag.sum() == 8


def test_oracle_coplanar_faces_smaller_index_wins(host):
    for order in ((0, 1), (1, 0)):
        tris = [[(0, 0), (9, 0), (0, 9)], [(2, 1), (10, 3), (3, 10)]]
        v, f = _screen_mesh([tris[k] for k in order])
        H = W = 12
        o = O.raster64(v, f, K1, R1, T1, H, W)
        both = o["cert"].numpy()
        z = o["z"].numpy()[both]
        np.testing.assert_array_equal(z, 1.0)            # one plane, z = 1 at every covered pair
        p2f, _ = brute(host, v, f, K1, R1, T1, H, W)
        cert_pix = o["pix"].numpy()[both]
        cnt = np.bincount(cert_pix, minlength=H * W).reshape(H, W)
        overlap = cnt == 2
        assert overlap.sum() > 10
        assert (p2f[0][overlap] == 0).all()              # equal depth: the smaller index
        assert not o["decided"].numpy()[overlap].any()   # a depth tie is never decided by the oracle
        assert O.admissible(o, torch.from_numpy(p2f[0]), len(f)).all()


def _cube():
    s = np.array([[x, y, z] for x in (-.5, .5) for y in (-.5, .5) for z in (-.5, .5)], np.float32)
    quads = [(0, 1, 3, 2), (4, 6, 7, 5), (0, 4, 5, 1), (2, 3, 7, 6), (0, 2, 6, 4), (1, 5, 7, 3)]
    f = np.array([t for q in quads for t in ((q[0], q[1], q[2]), (q[0], q[2], q[3]))], np.int32)
    return s, f


def test_oracle_unit_cube_at_a_known_pose(host):
    v, f = _cube()
    H = W = 64
    Km = np.array([[100, 0, 32], [0, 100, 32], [0, 0, 1]], np.float32)
    t = np.array([0, 0, 3], np.float32)                  # the face z = -0.5 at depth 2.5: the square [12, 52]^2
    o = O.raster64(v, f, Km, R1, t, H, W)
    front = np.nonzero((v[f][:, :, 2] == -0.5).all(1))[0]
    i, j = np.mgrid[0:H, 0:W]
    inner = (i >= 12) & (i <= 51) & (j >= 12) & (j <= 51)
    ans, dec = o["answer"].numpy(), o["decided"].numpy()
    clear = inner & (np.abs(i - j) > 1)                  # off the front face's diagonal
    assert dec[clear].all() and np.isin(ans[clear], front).all()
    assert dec[~inner].all() and (ans[~inner] == -1).all()
    cf = np.isin(o["face"].numpy(), front) & o["cert"].numpy()
    np.testing.assert_allclose(o["z"].numpy()[cf], 2.5, rtol=1e-12)
    p2f, st = brute(host, v, f, Km, R1, t, H, W)
    assert st == 0 and O.admissible(o, torch.from_numpy(p2f[0]), len(f)).all()
    assert np.array_equal(p2f[0][dec], ans[dec])


def test_faces_behind_and_across_the_camera(host):
    v = np.array([[0, 0, -1], [4, 0, -1], [0, 4, -1],            # behind: skipped, no status
                  [0, 0, 1], [8, 0, -1], [0, 8, 1],              # across z = 0: skipped, the near bit
                  [1, 1, 1], [6, 1, 1], [1, 6, 1]], np.float32)
    f = np.arange(9, dtype=np.int32).reshape(3, 3)
    o = O.raster64(v, f, K1, R1, T1, 10, 10)
    assert o["front_poss"].tolist() == [False, False, True]
    assert set(o["face"].tolist()) == {2}
    code, _, _, _ = pairs(host, v, f, K1, R1, T1, 10, 10, np.zeros(0), np.zeros(0), np.zeros(0))
    assert code.tolist() == [1, 2, 0]
    p2f, st = brute(host, v, f, K1, R1, T1, 10, 10)
    assert st == 8 and set(np.unique(p2f).tolist()) == {-1, 2}
    p2f, st = brute(host, v[:3], f[:1], K1, R1, T1, 10, 10)
    assert st == 0 and (p2f == -1).all()


# ---------------------------------------------------------------------------------------------- the host harness
MESHES = ["head", "head_holes", "degenerate", "big"]


def _view_cases(name, n_views, H, W, seed):
    v, f = K.MESHES[name]()
    Ks, Rs, ts = O.sphere_cameras(n_views, H, W, seed, radius=0.35 if name != "degenerate" else 0.4)
    return v, f, Ks, Rs, ts


def check_view(host, v, f, Km, Rm, tm, H, W, p2f=None):
    """Harness against the oracle in one view -> (largest |w - W| / E_W, largest depth error over its half-width)."""
    o = O.raster64(v, f, Km, Rm, tm, H, W)
    face, row, col = (o[k].numpy() for k in ("face", "row", "col"))
    code, w, cov, z = pairs(host, v, f, Km, Rm, tm, H, W, face, row, col)
    drawn = o["drawn_cert"].numpy()[face]
    W64, EW = o["W"].numpy(), o["EW"].numpy()
    err = np.abs(w.astype(np.float64) - W64)
    assert (err[drawn] <= EW[drawn]).all()
    cert, poss = o["cert"].numpy(), o["poss"].numpy()
    assert cov[cert].all() and not cov[~poss].any()
    zl, zh = o["z_lo"].numpy(), o["z_hi"].numpy()
    zc = z.astype(np.float64)
    assert ((zc[cert] >= zl[cert]) & (zc[cert] <= zh[cert])).all()
    if p2f is None:
        p2f, _ = brute(host, v, f, Km[None], Rm[None], tm[None], H, W)
        p2f = p2f[0]
    dec, ans = o["decided"].numpy(), o["answer"].numpy()
    assert np.array_equal(p2f[dec], ans[dec])
    assert O.admissible(o, torch.from_numpy(p2f), len(f)).all()
    with np.errstate(invalid="ignore"):
        half = np.maximum(zh - o["z"].numpy(), o["z"].numpy() - zl)
    r_w = (err[drawn] / EW[drawn]).max() if drawn.any() else 0.0
    r_z = (np.abs(zc - o["z"].numpy())[cert] / half[cert]).max() if cert.any() else 0.0
    return r_w, r_z, dec.mean()


@pytest.mark.parametrize("name", MESHES)
def test_harness_agrees_with_the_oracle(host, name):
    H, W = (72, 96) if name == "big" else (96, 128)
    v, f, Ks, Rs, ts = _view_cases(name, 2 if name == "big" else 4, H, W, 31)
    worst = np.zeros(3)
    for b in range(len(Ks)):
        r = check_view(host, v, f, Ks[b], Rs[b], ts[b], H, W)
        worst = np.maximum(worst, [r[0], r[1], 1 - r[2]])
    print(f"{name}: largest error / bound: edge functions {worst[0]:.3g}, depth {worst[1]:.3g}; "
          f"undecided pixels at most {worst[2]:.2%}")


# ------------------------------------------------------------------------------------ the script's visibility logic
def test_script_visibility_hand_cases():
    faces = np.array([[0, 1, 2], [1, 2, 3], [3, 4, 5], [4, 5, 0]], np.int32)
    V = 7                                                # vertex 6 belongs to no face: no view sees it
    p = np.array([
        [[-1, 0], [1, 1]],        # -1 present: [1:] drops it, faces {0, 1}
        [[2, 2], [3, 1]],         # every pixel covered: [1:] drops face 1 (the smallest), faces {2, 3}
        [[3, 3], [3, 3]],         # one face everywhere: [1:] leaves nothing
    ], np.int32)
    head = np.array([
        [[True, True], [True, False]],    # head variant [[-1, 0], [1, -1]]: faces {0, 1}
        [[True, True], [True, True]],     # head covers all: drops face 1 again -> {2, 3}
        [[False, False], [False, False]],  # empty head mask: nothing
    ])
    vis_mask, vm, vmh = O.script_visibility(p, head, faces, V)
    # view 0 sees faces {0,1}: verts {0,1,2,3}; view 1 faces {2,3}: verts {0,3,4,5}; view 2 nothing
    np.testing.assert_array_equal(vm, [2, 1, 1, 2, 1, 1, 0])
    np.testing.assert_array_equal(vmh, [2, 1, 1, 2, 1, 1, 0])
    assert vm.dtype == np.float32 and vmh.dtype == np.float32
    # head masks differing: view 0 head only over the face-0 pixel
    head2 = head.copy()
    head2[0] = [[False, True], [False, False]]    # [[-1, 0], [-1, -1]]: faces {0}: verts {0, 1, 2}
    vis_mask2, vm2, vmh2 = O.script_visibility(p, head2, faces, V)
    np.testing.assert_array_equal(vmh2, [2, 1, 1, 1, 1, 1, 0])
    with np.errstate(invalid="ignore"):
        prob = 1 - vmh2 / vm2
    assert np.isnan(prob[6])
    # vertex 3: prob_hair = 1 - 1/2 = 0.5, not > 0.5; seen by 2 of 3 views: False.  vertex 6: NaN, 0 / 3 < 0.1: True
    assert vis_mask2.tolist() == [False, False, False, False, False, False, True]
    assert vis_mask.tolist() == [False] * 6 + [True]
    # a vertex every view sees but never as head: prob_hair = 1 > 0.5
    _, vm3, vmh3 = O.script_visibility(p, np.zeros_like(head), faces, V)
    assert (vmh3 == 0).all()


def test_head_masks_equal_cv2_dilate_and_the_scripts_thresholds():
    cv2 = pytest.importorskip("cv2")
    from gaussianhaircut_b200.mesh import head_masks
    rng = np.random.default_rng(4)
    B, H, W = 3, 37, 53
    hair = np.zeros((B, H, W, 3), np.uint8)
    body = np.zeros((B, H, W, 3), np.uint8)
    for b in range(B):
        # sparse 0/255 masks and a few mid-grey values, with marks on every border row and column
        for m in (hair, body):
            m[b][rng.random((H, W)) < 0.03] = 255
            m[b][rng.random((H, W)) < 0.01] = rng.integers(100, 160)
            m[b][0, rng.integers(0, W)] = 255
            m[b][-1, rng.integers(0, W)] = 255
            m[b][rng.integers(0, H), 0] = 255
            m[b][rng.integers(0, H), -1] = 255
    got = head_masks(torch.from_numpy(hair), torch.from_numpy(body)).numpy()
    for b in range(B):
        mask_hair = cv2.dilate(hair[b], np.ones((5, 5))) / 255. >= 0.5
        mask = cv2.dilate(body[b], np.ones((5, 5))) / 255. >= 0.5
        mask_head = np.clip(mask.astype("float32") - mask_hair.astype("float32"), 0, 1)
        ref = mask_head[:, :, 0] >= 0.5
        assert np.array_equal(got[b], ref), b
    assert np.array_equal(head_masks(torch.from_numpy(hair[..., 0]), torch.from_numpy(body[..., 0])).numpy(), got)


# ------------------------------------------------------------------------------------------------------- the C ABI
def test_workspace_size_without_gpu(lib):
    from gaussianhaircut_b200 import _capi
    b = C.c_size_t()
    assert lib.gh_mesh_raster_workspace_size(5023, 9936, 1024, 1024, 16, C.byref(b)) == 0
    need = 16 * 1024 * 1024 * 8 + 16 * 9936 * 80 + 2 * 16 * 9936 + 2 * 16 * 5023 + 16 * 16
    assert need <= b.value <= need + 5 * 256
    bad = [(0, 10, 8, 8, 1, b"V and F"), (10, 0, 8, 8, 1, b"V and F"), (1 << 31, 10, 8, 8, 1, b"V and F"),
           (10, 10, 0, 8, 1, b"H and W"), (10, 10, 8, 8193, 1, b"H and W"), (10, 10, 8, 8, 0, b"chunk"),
           (10, 10, 8192, 8192, 32, b"chunk"), (10, 1 << 30, 8, 8, 2, b"chunk")]
    for V, F, H, W, ch, msg in bad:
        assert lib.gh_mesh_raster_workspace_size(V, F, H, W, ch, C.byref(b)) == _capi.GH_E_INVALID_ARG
        assert msg in lib.gh_last_error(), (msg, lib.gh_last_error())
    assert lib.gh_mesh_raster_workspace_size(10, 10, 8, 8, 1, None) == _capi.GH_E_INVALID_ARG


def test_entry_point_refuses_bad_arguments_before_any_launch(lib):
    from gaussianhaircut_b200 import _capi
    p = lambda x: C.c_void_p(x)  # noqa: E731
    V, F, H, W, ch = 10, 20, 8, 8, 2
    nb = C.c_size_t()
    lib.gh_mesh_raster_workspace_size(V, F, H, W, ch, C.byref(nb))
    nb = nb.value
    base = dict(V=V, F=F, verts=p(0x10000), faces=p(0x20000), B=3, K=p(0x30000), R=p(0x40000), t=p(0x50000), H=H, W=W,
                head=None, p2f=p(0x60000), vis=None, c0=None, c1=None, chunk=ch, ws=p(0x100000), bytes=nb,
                status=p(0x70000), debug=0)
    order = list(base)

    def call(**kw):
        a = dict(base, **kw)
        return lib.gh_mesh_raster(*[a[k] for k in order], None)

    cases = [
        (dict(V=0), b"V and F"), (dict(F=1 << 31), b"V and F"), (dict(H=0), b"H and W"), (dict(W=9000), b"H and W"),
        (dict(chunk=0), b"chunk"), (dict(B=0), b"B must be"), (dict(verts=None), b"missing verts"),
        (dict(faces=None), b"missing verts"), (dict(K=None), b"missing verts"), (dict(R=None), b"missing verts"),
        (dict(t=None), b"missing verts"), (dict(status=None), b"missing verts"),
        (dict(verts=p(0x10002)), b"4-byte aligned"), (dict(p2f=p(0x60001)), b"4-byte aligned"),
        (dict(c0=p(0x80000)), b"go together"), (dict(c1=p(0x80000)), b"go together"),
        (dict(p2f=None), b"no output"), (dict(ws=None), b"missing workspace"),
        (dict(ws=p(0x100080)), b"256-byte aligned"), (dict(bytes=nb - 1), b"workspace of"),
    ]
    n0 = lib.gh_kernel_launch_count()
    for kw, msg in cases:
        assert call(**kw) == _capi.GH_E_INVALID_ARG, msg
        assert msg in lib.gh_last_error(), (msg, lib.gh_last_error())
    lib.gh_stage_timing_enable(1)
    try:
        assert call(debug=1) == _capi.GH_E_INVALID_ARG
        assert b"stage timer" in lib.gh_last_error()
    finally:
        lib.gh_stage_timing_enable(0)
    assert lib.gh_kernel_launch_count() == n0


def test_python_refusals_need_no_gpu():
    from gaussianhaircut_b200 import mesh as M
    v = torch.zeros(3, 3)
    f = torch.tensor([[0, 1, 2]], dtype=torch.int32)
    Km, Rm, tm = torch.eye(3)[None], torch.eye(3)[None], torch.zeros(1, 3)
    with pytest.raises(RuntimeError, match="CUDA tensors"):
        M.rasterize_faces(v, f, Km, Rm, tm, 8, 8)
    with pytest.raises(RuntimeError, match="Int"):
        M.rasterize_faces(v, f.long(), Km, Rm, tm, 8, 8)
    with pytest.raises(RuntimeError, match="'t' must have shape"):
        M.rasterize_faces(v, f, Km, Rm, torch.zeros(2, 3), 8, 8)
    with pytest.raises(RuntimeError, match="H and W"):
        M.rasterize_faces(v, f, Km, Rm, tm, 0, 8)
    with pytest.raises(RuntimeError, match="bool"):
        M.scalp_visibility(v, f, Km, Rm, tm, torch.zeros(1, 8, 8, dtype=torch.uint8))
    with pytest.raises(RuntimeError, match="head masks for K"):
        M.scalp_visibility(v, f, Km, Rm, tm, torch.zeros(2, 8, 8, dtype=torch.bool))
    with pytest.raises(RuntimeError, match="uint8"):
        M.head_masks(torch.zeros(1, 8, 8), torch.zeros(1, 8, 8))
    with pytest.raises(RuntimeError, match="differ in shape"):
        M.head_masks(torch.zeros(1, 8, 8, dtype=torch.uint8), torch.zeros(1, 8, 9, dtype=torch.uint8))
