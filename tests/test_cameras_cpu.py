"""CPU tests of the trainable cameras (DESIGN §17):

  * the camera model of csrc/gh_camera_math.h, compiled for the host (tests/host_harness/camera_host.cpp), against a
    float64 restatement of the reference's chain (forward within float32 rounding, backward against float64 autograd)
    and against the reference's own `lie.se3_to_SE3` evaluated on the CPU, at rotation angles 0, 1e-6, 0.3, 2 and 3,
    tiny and large translations, FoV residuals of +-0.2 and the row without intrinsics;
  * the camera entry points of the C ABI refuse bad arguments before they launch anything;
  * CameraRig.reference_dicts() / write_back() round-trip, the configurations the rig rejects, and the capture key of
    graphs.CapturedTrainStep changing with the rig's storage and with train_cameras.
"""
import ctypes as C
import math
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

import _util

ROOT = _util.ROOT
HARNESS_SRC = os.path.join(ROOT, "tests", "host_harness", "camera_host.cpp")
HARNESS_SO = os.path.join(ROOT, "tests", "host_harness", "libcamera_host.so")
MATH_H = os.path.join(ROOT, "gaussianhaircut_b200", "csrc", "gh_camera_math.h")
EPS32 = float(np.finfo(np.float32).eps)


@pytest.fixture(scope="module")
def host():
    newest = max(os.path.getmtime(HARNESS_SRC), os.path.getmtime(MATH_H))
    if not os.path.isfile(HARNESS_SO) or os.path.getmtime(HARNESS_SO) < newest:
        subprocess.run(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-std=c++17", "-w", HARNESS_SRC, "-o",
                        HARNESS_SO], check=True)
    h = C.CDLL(HARNESS_SO)
    h.gh_host_camera_forward.argtypes = [C.c_int] + [C.c_void_p] * 6
    h.gh_host_camera_forward.restype = None
    h.gh_host_camera_backward.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
    h.gh_host_camera_backward.restype = None
    return h


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def host_forward(h, base, r):
    n = base.shape[0]
    base, r = np.ascontiguousarray(base, np.float32), np.ascontiguousarray(r, np.float32)
    v, p, c, t = (np.zeros((n, k), np.float32) for k in (16, 16, 3, 2))
    h.gh_host_camera_forward(n, _p(base), _p(r), _p(v), _p(p), _p(c), _p(t))
    return v.reshape(n, 4, 4), p.reshape(n, 4, 4), c, t


def host_backward(h, base, r, g, intrinsics=1):
    n = base.shape[0]
    base, r, g = (np.ascontiguousarray(a, np.float32) for a in (base, r, g))
    dr = np.zeros((n, 8), np.float32)
    h.gh_host_camera_backward(n, _p(base), _p(r), _p(g), int(intrinsics), _p(dr))
    return dr


# --------------------------------------------------------------------------------------------- float64 restatement
def _den(k, i):
    d = 1.0
    for j in range(i + 1):
        if k == 0:
            d *= (2 * j) * (2 * j + 1) if j > 0 else 1
        elif k == 1:
            d *= (2 * j + 1) * (2 * j + 2)
        else:
            d *= (2 * j + 2) * (2 * j + 3)
    return d


def restate(base, r):
    """The reference chain (cameras.py:95-152, camera_opt_utils.py:84-141, graphics_utils.py:51) in float64 torch:
    base (18,), r (8,) -> viewmatrix, projmatrix, campos, tan_fov.  Differentiable in r."""
    w, u, f = r[:3], r[3:6], r[6:8]
    z = torch.zeros((), dtype=torch.float64)
    K = torch.stack([torch.stack([z, -w[2], w[1]]), torch.stack([w[2], z, -w[0]]), torch.stack([-w[1], w[0], z])])
    s = (w * w).sum()
    A, B, Cc = (sum((-1) ** i * s ** i / _den(k, i) for i in range(11)) for k in range(3))
    I = torch.eye(3, dtype=torch.float64)
    R = I + A * K + B * (K @ K)
    V = I + B * K + Cc * (K @ K)
    Res = torch.cat([torch.cat([R, (V @ u)[:, None]], 1), torch.tensor([[0.0, 0.0, 0.0, 1.0]], dtype=torch.float64)], 0)
    W = (base[:16].reshape(4, 4) @ Res).T
    tan = torch.tan((base[16:18] + f) / 2)
    znear, zfar = 0.01, 100.0
    top, right = tan[1] * znear, tan[0] * znear
    P = torch.zeros(4, 4, dtype=torch.float64)
    P = P.index_put((torch.tensor([0]), torch.tensor([0])), (2 * znear / (2 * right)).reshape(1))
    P = P.index_put((torch.tensor([1]), torch.tensor([1])), (2 * znear / (2 * top)).reshape(1))
    P[3, 2] = 1.0
    P[2, 2] = zfar / (zfar - znear)
    P[2, 3] = -(zfar * znear) / (zfar - znear)
    full = W @ P.T
    campos = torch.linalg.inv(W)[3, :3]
    return W, full, campos, tan


def _rot(axis, ang):
    a = np.asarray(axis, np.float64)
    return a / np.linalg.norm(a) * ang


def _colmap(seed):
    """A float32 world-to-camera matrix like getWorld2View2's: a rotation and a translation of a few units."""
    g = np.random.default_rng(seed)
    q, _ = np.linalg.qr(g.normal(size=(3, 3)))
    if np.linalg.det(q) < 0:
        q[:, 0] *= -1
    M = np.eye(4)
    M[:3, :3], M[:3, 3] = q, g.normal(size=3) * 2.5
    return M.astype(np.float32)


def _cases():
    out = []
    for k, theta in enumerate((0.0, 1e-6, 0.3, 2.0, 3.0)):
        for t_scale in (1e-7, 0.05, 30.0):
            for f in ((0.0, 0.0), (0.2, -0.2), (-0.2, 0.2)):
                w = _rot((1.0, -2.0 + k, 0.5), theta) if theta else np.zeros(3)
                u = np.array([0.3, -1.0, 0.7]) * t_scale
                base = np.concatenate([_colmap(k).reshape(16), [0.9 + 0.1 * k, 0.7 + 0.05 * k]])
                out.append((base.astype(np.float32), np.concatenate([w, u, f]).astype(np.float32)))
    return out


CASES = _cases()


def test_forward_matches_float64(host):
    base = np.stack([b for b, _ in CASES])
    r = np.stack([x for _, x in CASES])
    v, p, c, t = host_forward(host, base, r)
    for i, (b, x) in enumerate(CASES):
        ref = [a.detach().numpy() for a in restate(torch.tensor(b, dtype=torch.float64), torch.tensor(x, dtype=torch.float64))]
        for got, want, name in zip((v[i], p[i], c[i], t[i]), ref, ("view", "proj", "campos", "tan")):
            scale = max(1.0, float(np.abs(want).max()))
            err = float(np.abs(got.astype(np.float64) - want).max())
            # a few roundings per entry of magnitude <= scale; campos: the inverse of a float32 matrix of norm ~|t|
            bound = (64 if name == "campos" else 16) * EPS32 * scale
            assert err <= bound, (i, name, err, bound)


def _upstream(seed, n, full):
    g = np.random.default_rng(seed).normal(size=(n, 37)).astype(np.float32)
    if not full:
        # the entries the projection backward never writes (include/gh_rasterizer.h: d_camera) are zero
        g[:, [3, 7, 11, 15, 18, 22, 26, 30]] = 0
    return g


@pytest.mark.parametrize("full", [False, True], ids=["projection-layout", "all-37"])
@pytest.mark.parametrize("intrinsics", [1, 0])
def test_backward_matches_float64_autograd(host, intrinsics, full):
    base = np.stack([b for b, _ in CASES])
    r = np.stack([x for _, x in CASES])
    if not intrinsics:
        r[:, 6:] = 0
    g = _upstream(3, len(CASES), full)
    dr = host_backward(host, base, r, g, intrinsics)
    worst = 0.0
    for i in range(len(CASES)):
        rr = torch.tensor(r[i], dtype=torch.float64, requires_grad=True)
        outs = restate(torch.tensor(base[i], dtype=torch.float64), rr)
        gi = torch.tensor(g[i], dtype=torch.float64)
        L = (outs[0].reshape(-1) * gi[:16]).sum() + (outs[1].reshape(-1) * gi[16:32]).sum() + \
            (outs[2] * gi[32:35]).sum() + (outs[3] * gi[35:37]).sum()
        want = torch.autograd.grad(L, rr)[0].numpy()
        if not intrinsics:
            want[6:] = 0
        scale = max(1e-30, float(np.abs(want).max()))
        err = float(np.abs(dr[i].astype(np.float64) - want).max()) / scale
        worst = max(worst, err)
        assert err <= 1e-6, (i, err, dr[i], want)
    assert np.isfinite(dr).all()


def _ref_lie():
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import ref_python
    src = ref_python.ref_src_dir()
    if src is None or not os.path.isfile(os.path.join(src, "utils", "camera_opt_utils.py")):
        pytest.skip("the reference's Python sources are not available")
    ref_python.install_stubs()
    if src not in sys.path:
        sys.path.insert(0, src)
    from utils.camera_opt_utils import lie
    return lie


def test_se3_matches_reference_lie(host):
    lie = _ref_lie()
    rows = np.stack([x for _, x in CASES])
    base = np.zeros((len(CASES), 18), np.float32)
    base[:, :16] = np.eye(4, dtype=np.float32).reshape(16)
    base[:, 16:] = 1.0
    v, _, _, _ = host_forward(host, base, rows)
    want = lie.se3_to_SE3(torch.tensor(rows[:, :6])).numpy()      # (n, 3, 4), float32 on the CPU
    got = v.transpose(0, 2, 1)[:, :3, :]                             # viewmatrix = Res^T with C = I
    for i in range(len(CASES)):
        scale = max(1.0, float(np.abs(want[i]).max()))
        assert float(np.abs(got[i] - want[i]).max()) <= 16 * EPS32 * scale, i


# --------------------------------------------------------------------------------------------- C ABI refusals
@pytest.fixture(scope="module")
def lib():
    from gaussianhaircut_b200 import _capi
    return _capi.load()


F = C.c_void_p(4096)        # never dereferenced: every call below is refused on the host
ODD = C.c_void_p(4097)


def _fwd(lib, n=4, debug=0, residuals=F, status=F):
    return lib.gh_camera_forward(n, residuals, F, F, F, F, F, F, status, debug, None)


def _bwd(lib, n=4, debug=0, d_camera=F, nan=F):
    return lib.gh_camera_backward(n, F, F, F, 1, d_camera, F, F, nan, F, debug, None)


def _adam(lib, n=4, debug=0, lrs=F, skip=None):
    return lib.gh_camera_adam_step(n, 1, F, F, F, F, F, F, lrs, 0.9, 0.999, 1e-15, F, skip, debug, None)


def test_camera_abi_refusals(lib):
    from gaussianhaircut_b200 import _capi
    n0 = lib.gh_kernel_launch_count()
    cases = [
        (lambda: _fwd(lib, n=0), "n must be positive"), (lambda: _fwd(lib, residuals=None), "missing"),
        (lambda: _fwd(lib, status=None), "missing"), (lambda: _fwd(lib, residuals=ODD), "aligned"),
        (lambda: _fwd(lib, debug=1), "debug"),
        (lambda: _bwd(lib, n=-1), "n must be positive"), (lambda: _bwd(lib, d_camera=None), "missing"),
        (lambda: _bwd(lib, nan=ODD), "aligned"), (lambda: _bwd(lib, debug=1), "debug"),
        (lambda: _adam(lib, n=0), "n must be positive"), (lambda: _adam(lib, lrs=None), "missing"),
        (lambda: _adam(lib, skip=ODD), "aligned"), (lambda: _adam(lib, debug=1), "debug"),
    ]
    for call, msg in cases:
        assert call() == _capi.GH_E_INVALID_ARG
        assert msg in lib.gh_last_error().decode()
    lib.gh_stage_timing_enable(1)
    try:
        assert _fwd(lib) == _capi.GH_E_INVALID_ARG and "stage timer" in lib.gh_last_error().decode()
    finally:
        lib.gh_stage_timing_enable(0)
    assert lib.gh_kernel_launch_count() == n0


# --------------------------------------------------------------------------------------------- Python layer
def _ref_like_camera(k, fov=True):
    cam = types.SimpleNamespace(image_name=f"img_{k:03d}", image_width=64 + k, image_height=48,
                                _colmap_transform=torch.tensor(_colmap(k)), _FoVx=torch.tensor([0.9]), _FoVy=torch.tensor([0.7]),
                                _rotation_res=torch.nn.Parameter(torch.randn(3)),
                                _translation_res=torch.nn.Parameter(torch.randn(3)))
    if fov:
        cam._fov_res = torch.nn.Parameter(torch.randn(2))
    return cam


def test_reference_dicts_write_back_round_trip():
    from gaussianhaircut_b200.cameras import CameraRig
    cams = [_ref_like_camera(k) for k in range(3)]
    rig = CameraRig.from_cameras(cams)
    rot, trans, fov = rig.reference_dicts()
    assert list(rot) == [c.image_name for c in cams]
    for c in cams:
        assert torch.equal(rot[c.image_name], c._rotation_res.detach())
        assert torch.equal(trans[c.image_name], c._translation_res.detach())
        assert torch.equal(fov[c.image_name], c._fov_res.detach())
    with torch.no_grad():
        rig.residuals.add_(0.125)
    rig.write_back(cams)
    for i, c in enumerate(cams):
        assert isinstance(c._rotation_res, torch.nn.Parameter)
        assert torch.equal(torch.cat([c._rotation_res, c._translation_res, c._fov_res]).detach(), rig.residuals.detach()[i])
    assert torch.equal(CameraRig.from_cameras(cams).residuals.detach(), rig.residuals.detach())
    # without intrinsics the fov dict is empty and f stays 0
    rig2 = CameraRig.from_cameras([_ref_like_camera(0, fov=False)], intrinsics=False)
    assert rig2.reference_dicts()[2] == {} and torch.count_nonzero(rig2.residuals.detach()[:, 6:]) == 0
    with pytest.raises(RuntimeError, match="CUDA"):
        rig2.forward(rig2.indices[:1])


def test_rejected_configurations():
    from gaussianhaircut_b200.cameras import CameraRig
    c = _ref_like_camera(0)
    c.use_barf = False
    c._rotation_res = torch.nn.Parameter(torch.eye(3)[:2].reshape(-1).clone())
    with pytest.raises(ValueError, match="use_barf=True"):
        CameraRig.from_cameras([c])
    c = _ref_like_camera(0)
    c.trainable_cameras, c.trainable_intrinsics = False, True
    with pytest.raises(ValueError, match="without trainable cameras"):
        CameraRig.from_cameras([c])
    with pytest.raises(ValueError, match="_fov_res"):
        CameraRig.from_cameras([_ref_like_camera(0, fov=False)])
    # a trained field of view must not be dropped: intrinsics=False with a trainable or non-zero _fov_res
    c = _ref_like_camera(0)
    with pytest.raises(ValueError, match="intrinsics=False"):
        CameraRig.from_cameras([c], intrinsics=False)
    c._fov_res = torch.nn.Parameter(torch.zeros(2))
    c.trainable_intrinsics = True
    with pytest.raises(ValueError, match="intrinsics=False"):
        CameraRig.from_cameras([c], intrinsics=False)
    c.trainable_intrinsics = False
    assert CameraRig.from_cameras([c], intrinsics=False).n == 1


def test_capture_key_tracks_rig_and_train_flag():
    from gaussianhaircut_b200.cameras import CameraAdam, CameraRig
    from gaussianhaircut_b200.graphs import capture_key
    params = [torch.zeros(16, 3)]
    model = types.SimpleNamespace(_xyz=params[0], active_sh_degree=3, xyz_gradient_accum=torch.zeros(16, 1),
                                  denom=torch.zeros(16, 1), max_radii2D=torch.zeros(16))
    opt = types.SimpleNamespace(param_groups=[{"params": params}], state={})
    rig = CameraRig.from_cameras([_ref_like_camera(k) for k in range(2)])
    cam_opt = CameraAdam(rig, 1e-3, 1e-3, 1e-3, capturable=True)
    k = capture_key(model, opt, 64, 48, rig, cam_opt, True)
    assert capture_key(model, opt, 64, 48, rig, cam_opt, True) == k
    assert capture_key(model, opt, 64, 48, rig, cam_opt, False) != k
    assert capture_key(model, opt, 64, 48) != k
    rig.grad = torch.zeros_like(rig.grad)
    assert capture_key(model, opt, 64, 48, rig, cam_opt, True) != k
    k = capture_key(model, opt, 64, 48, rig, cam_opt, True)
    cam_opt.exp_avg = torch.zeros_like(cam_opt.exp_avg)
    assert capture_key(model, opt, 64, 48, rig, cam_opt, True) != k
