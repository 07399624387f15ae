"""Strand model rendered from its polylines (render_hair_strands), without a GPU.

* the restated strand geometry (tests/_strands.py `strand_geometry_reference` + oracle/synth.py `project_reference`)
  against the reference's own GaussianModelCurves running its own initialize_gaussians_hair()
  (tests/golden/pyref_strands.npz, make_golden_pyref_strands.py): values and every gradient incl. the camera;
* the strand instantiation of the product's per-Gaussian arithmetic (gh_project_math.h with STRAND = true, compiled
  for the host by tests/host_harness/strand_host.cpp) against autograd of that restatement: values, the folded
  segment-vector term and the midpoint term of the backward, the camera gradients;
* the flag encoding: bit 10 selects the strand instantiation, the existing configurations encode as before;
* the strand-mode argument checks of the C entry points (they run before any device work).
The midpoint and suffix-sum kernels run on the GPU only: tests/test_gpu_strands.py."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import _strands  # noqa: E402
import _util  # noqa: E402

synth = _util.synth
HARNESS_SRC = os.path.join(ROOT, "tests", "host_harness", "strand_host.cpp")
HARNESS_SO = os.path.join(ROOT, "tests", "host_harness", "libstrand_host.so")
MATH_H = os.path.join(ROOT, "gaussianhaircut_b200", "csrc", "gh_project_math.h")
GOLDEN = os.path.join(ROOT, "tests", "golden", "pyref_strands.npz")


def _rel(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    nb = b.norm().item()
    return (a - b).norm().item() / nb if nb > 0 else (a - b).norm().item()


def test_strand_flag_is_bit_10_and_the_existing_configurations_are_unchanged():
    from gaussianhaircut_b200 import projection as pj
    assert pj.encode_flags(pj.HAIR_STRANDS) == pj.encode_flags(pj.HAIR_MODEL) | (1 << 10)
    for cfg in (pj.GAUSSIAN_MODEL, pj.HAIR_MODEL, pj.HEAD_PRECOMP):
        assert pj.encode_flags(cfg) < (1 << 10)
    assert {k: v for k, v in pj.HAIR_STRANDS.items() if k != "strands"} == pj.HAIR_MODEL


# ------------------------------------------------------------------ restatement pinned on the reference's own class
def _camera(d, grad=True):
    cam = dict(synth.make_camera(int(d["cam_k"]), int(d["W"]), int(d["H"])))
    if grad:
        for k in ("world_view_transform", "full_proj_transform", "camera_center"):
            cam[k] = cam[k].clone().requires_grad_(True)
    return cam


@pytest.mark.parametrize("model", ["s6_l33", "s4_l99"])
def test_strand_restatement_matches_the_reference_model(model):
    d = np.load(GOLDEN)
    g = lambda k: torch.from_numpy(d[f"{model}/{k}"])  # noqa: E731
    S, L, seed = int(g("S")), int(g("L")), int(g("seed"))
    poly = _strands.make_strand_polylines(S, L, seed)
    leaves = {k: poly[k].clone().requires_grad_(True) for k in ("dirs", "f_dc", "f_rest", "conf")}
    cam = _camera(d)
    ref, geo = _strands.project_strands_reference(poly["origins"], leaves["dirs"], poly["scale"], leaves["f_dc"],
                                                  leaves["f_rest"], leaves["conf"], cam)
    assert torch.equal(ref["mask"], g("mask"))
    for k in ("xyz", "scaling", "rotation"):
        assert _rel(geo[k].detach(), g(k)) <= 1e-5, k
    for k in ("means2D", "conic", "colors"):
        assert _rel(ref[k].detach(), g(k)) <= 1e-5, f"{k}: {_rel(ref[k].detach(), g(k))}"
    m = ref["mask"][:, None].float()
    sum((ref[k] * g("W_" + k) * m).sum() for k in ("conic", "means2D", "colors")).backward()
    for k, t in leaves.items():
        assert _rel(t.grad, g("g_" + k)) <= 1e-4, f"{k}: {_rel(t.grad, g('g_' + k))}"
    assert _rel(cam["world_view_transform"].grad, g("g_viewmatrix")) <= 1e-4
    assert _rel(cam["full_proj_transform"].grad, g("g_projmatrix")) <= 1e-4
    assert _rel(cam["camera_center"].grad, g("g_campos")) <= 1e-4


# ------------------------------------------------------------------ host build of the strand instantiation
@pytest.fixture(scope="module")
def host():
    newest = max(os.path.getmtime(HARNESS_SRC), os.path.getmtime(MATH_H))
    if not os.path.isfile(HARNESS_SO) or os.path.getmtime(HARNESS_SO) < newest:
        subprocess.run(["g++", "-O2", "-shared", "-fPIC", "-std=c++17", "-w", HARNESS_SRC, "-o", HARNESS_SO], check=True)
    return C.CDLL(HARNESS_SO)


def _p(t):
    return C.c_void_p(t.data_ptr())


def _host_run(host, xyz, dirs, scale, f_dc, f_rest, conf, cam, sh_degree, mod, gin):
    from gaussianhaircut_b200 import projection as pj
    P = xyz.shape[0]
    c = lambda t: t.detach().contiguous().float()  # noqa: E731
    t = [c(xyz), torch.tensor([float(scale)]), c(dirs), c(f_dc), c(f_rest), c(conf)]
    V, Pm, cc = (c(cam[k]) for k in ("world_view_transform", "full_proj_transform", "camera_center"))
    common = (P, cam["image_width"], cam["image_height"], *(_p(x) for x in t), _p(V), _p(Pm), _p(cc),
              C.c_float(float(cam["tanfovx"])), C.c_float(float(cam["tanfovy"])), C.c_float(mod), sh_degree,
              C.c_uint(pj.encode_flags(pj.HAIR_STRANDS)), C.c_float(pj.HAIR_STRANDS["det_eps"]))
    out = {"means2D": torch.zeros(P, 3), "colors": torch.zeros(P, 10), "opacity": torch.zeros(P, 1), "conic": torch.zeros(P, 3),
           "cov3D": torch.zeros(P, 6), "mask": torch.zeros(P, dtype=torch.uint8)}
    host.gh_host_strand_forward(*common, *(_p(out[k]) for k in ("means2D", "colors", "opacity", "conic", "cov3D", "mask")))
    g = {k: c(v) for k, v in gin.items()}
    d = {"xyz": torch.zeros(P, 3), "dirs": torch.zeros(P, 3), "f_dc": torch.zeros(P, 1, 3), "f_rest": torch.zeros(P, 15, 3),
         "conf": torch.zeros(P, 1), "scaling_rotation": torch.ones(P, 7)}
    cam29 = np.zeros(29, dtype=np.float64)
    host.gh_host_strand_backward(*common, _p(out["mask"]), _p(g["means2D"]), _p(g["conic"]), _p(g["colors"]),
                                 *(_p(d[k]) for k in ("xyz", "dirs", "f_dc", "f_rest", "conf", "scaling_rotation")),
                                 cam29.ctypes.data_as(C.c_void_p))
    dV = np.zeros((4, 4)); dPm = np.zeros((4, 4))
    dV[:, :3] = cam29[:12].reshape(4, 3)
    dPm[:, [0, 1, 3]] = cam29[12:24].reshape(4, 3)
    d.update(viewmatrix=torch.from_numpy(dV), projmatrix=torch.from_numpy(dPm), campos=torch.from_numpy(cam29[24:27]),
             tan=torch.from_numpy(cam29[27:29]))
    return out, d


# case: (S, L, sh_degree, scaling modifier, camera tweak, segment lengths)
HOST_CASES = [
    (6, 33, 3, 1.0, None, None),
    (4, 99, 2, 0.8, None, None),
    (5, 40, 3, 1.0, None, "spread"),          # |d| from 1e-4 to 1e-2
    (6, 33, 3, 1.0, "narrow", None),          # narrow field of view: the +-1.3 tan(fov) clamp is active, some culled
]


@pytest.mark.parametrize("S,L,deg,mod,tweak,lengths", HOST_CASES)
def test_strand_projection_math_matches_autograd(host, S, L, deg, mod, tweak, lengths):
    poly = _strands.make_strand_polylines(S, L, seed=21)
    dirs = poly["dirs"]
    if lengths == "spread":
        g = torch.Generator().manual_seed(5)
        target = 10.0 ** (-4.0 + 2.0 * torch.rand(S, L, 1, generator=g))
        dirs = dirs / dirs.norm(dim=-1, keepdim=True) * target
    W, H = 200, 120
    cam = dict(synth.make_camera(7, W, H, focal_factor=(6.0 if tweak == "narrow" else 1.2)))
    camg = dict(cam)
    for k in ("world_view_transform", "full_proj_transform", "camera_center"):
        camg[k] = cam[k].clone().requires_grad_(True)
    camg["tanfovx"] = torch.tensor(cam["tanfovx"], dtype=torch.float32, requires_grad=True)
    camg["tanfovy"] = torch.tensor(cam["tanfovy"], dtype=torch.float32, requires_grad=True)
    # the midpoints enter the per-Gaussian arithmetic as their own leaf: the kernels see them as an input buffer
    geo = _strands.strand_geometry_reference(poly["origins"], dirs, poly["scale"])
    xyz = geo["xyz"].detach().clone().requires_grad_(True)
    dl = dirs.reshape(-1, 3).clone().requires_grad_(True)
    f = {k: poly[k].clone().requires_grad_(True) for k in ("f_dc", "f_rest", "conf")}
    loc = _strands.strand_geometry_reference(torch.zeros(S * L, 1, 3), dl[:, None, :], poly["scale"])
    raw = {"xyz": xyz, "scaling": loc["scaling"], "rotation": loc["rotation"], "dirs": dl, **f}
    ref = synth.project_reference(raw, camg, dict(synth.PROJECT_HAIR_MODEL), sh_degree=deg, scaling_modifier=mod)
    mask = ref["mask"]
    assert 0 < int(mask.sum())
    if tweak == "narrow":
        assert int(mask.sum()) < mask.numel()
    gg = torch.Generator().manual_seed(2)
    gin = {"means2D": torch.randn(ref["means2D"].shape, generator=gg), "conic": torch.randn(ref["conic"].shape, generator=gg) * 1e-3,
           "colors": torch.randn(ref["colors"].shape, generator=gg)}
    gin["means2D"][:, 2] = 0.0
    out, d = _host_run(host, xyz, dl, poly["scale"], f["f_dc"], f["f_rest"], f["conf"], cam, deg, mod, gin)
    assert torch.equal(out["mask"].bool(), mask)
    assert _rel(out["means2D"], ref["means2D"].detach()) <= 1e-5
    assert _rel(out["conic"][mask], ref["conic"].detach()[mask]) <= 1e-5
    assert _rel(out["colors"], ref["colors"].detach()) <= 1e-5
    assert _rel(out["cov3D"], ref["cov3D"].detach()) <= 1e-5
    assert float((out["opacity"] - 1.0).abs().max()) == 0.0
    m = mask[:, None].float()
    sum((ref[k] * gin[k] * m).sum() for k in gin).backward()
    assert float(d["scaling_rotation"].abs().max()) == 0.0          # folded into dirs, never written
    for k, src in (("dirs", dl), ("xyz", xyz), ("f_dc", f["f_dc"]), ("f_rest", f["f_rest"]), ("conf", f["conf"])):
        e = _rel(d[k].reshape(src.grad.shape), src.grad)
        assert e <= 2e-4, f"{k}: {e}"
        assert float(d[k].reshape(src.grad.shape)[~mask].abs().sum()) == 0.0, f"{k}: culled rows must be zero"
    assert _rel(d["viewmatrix"], camg["world_view_transform"].grad) <= 2e-4
    assert _rel(d["projmatrix"], camg["full_proj_transform"].grad) <= 2e-4
    assert _rel(d["campos"], camg["camera_center"].grad) <= 2e-4
    assert _rel(d["tan"], torch.stack([camg["tanfovx"].grad, camg["tanfovy"].grad])) <= 2e-4


# ------------------------------------------------------------------ strand-mode argument validation (no GPU needed)
def _lib():
    from gaussianhaircut_b200 import _capi
    return _capi.load(), _capi


def _proj_call(lib, which, flags, rotation=True, dirs=True, scaling=True, d_scaling=False, d_rotation=False, d_dirs=True):
    """One call of a projection entry point with dummy device addresses: every check runs before any device work."""
    fake = C.c_void_p(4096)
    nz = lambda on: fake if on else None  # noqa: E731
    common = (128, 64, 48, fake, nz(scaling), nz(rotation), nz(dirs), fake, fake, None, None, fake, fake, fake, fake,
              0.5, 0.5, 1.0, 3, flags, 1e-7)
    if which == "forward":
        return lib.gh_project_forward(*common, fake, fake, fake, fake, None, fake, None)
    if which == "binned":
        n, m = C.c_int(0), C.c_int(0)
        return lib.gh_project_forward_binned(*common, fake, fake, fake, fake, None, fake, fake, fake, fake, None, 0,
                                             C.byref(n), C.byref(m), None, None)
    return lib.gh_project_backward(*common, fake, None, fake, fake, fake, fake, fake, nz(d_scaling), nz(d_rotation), nz(d_dirs),
                                   fake, fake, None, None, fake, None, None, None, None, None)


@pytest.mark.parametrize("which", ["forward", "binned", "backward"])
def test_strand_mode_argument_errors(which):
    from gaussianhaircut_b200 import projection as pj
    lib, capi = _lib()
    strand = pj.encode_flags(pj.HAIR_STRANDS)
    cases = [
        (dict(rotation=True), "rotation must be NULL"),
        (dict(rotation=False, dirs=False), "needs dirs"),
        (dict(rotation=False, scaling=False), "strand thickness"),
    ]
    for kw, msg in cases:
        assert _proj_call(lib, which, strand, **kw) == capi.GH_E_INVALID_ARG, (which, kw)
        assert msg in lib.gh_last_error().decode(), (which, kw, lib.gh_last_error())
    for bad in (pj.encode_flags(dict(pj.HAIR_STRANDS, scale_act=1)), pj.encode_flags(dict(pj.HAIR_STRANDS, dir_mode=0))):
        assert _proj_call(lib, which, bad, rotation=False) == capi.GH_E_INVALID_ARG
        assert "scale activation 0 and direction mode 1" in lib.gh_last_error().decode()
    if which == "backward":
        for kw in (dict(d_scaling=True), dict(d_rotation=True)):
            assert _proj_call(lib, which, strand, rotation=False, **kw) == capi.GH_E_INVALID_ARG
            assert "d_scaling / d_rotation must be NULL" in lib.gh_last_error().decode()
        assert _proj_call(lib, which, strand, rotation=False, d_dirs=False) == capi.GH_E_INVALID_ARG
        assert "needs d_dirs" in lib.gh_last_error().decode()
    # the existing configurations keep their own checks: a missing rotation is still a missing mandatory pointer
    assert _proj_call(lib, which, pj.encode_flags(pj.HAIR_MODEL), rotation=False) == capi.GH_E_INVALID_ARG
    assert "missing mandatory pointer" in lib.gh_last_error().decode()


def test_strand_geometry_entry_point_errors():
    lib, capi = _lib()
    fake = C.c_void_p(4096)
    assert lib.gh_strand_midpoints(0, 5, fake, fake, fake, None) == capi.GH_E_INVALID_ARG
    assert "S and L must be positive" in lib.gh_last_error().decode()
    assert lib.gh_strand_midpoints(4, 5, None, fake, fake, None) == capi.GH_E_INVALID_ARG
    assert lib.gh_strand_backward(4, 0, fake, fake, None, None) == capi.GH_E_INVALID_ARG
    assert lib.gh_strand_backward(4, 5, fake, None, None, None) == capi.GH_E_INVALID_ARG
    assert "missing pointer" in lib.gh_last_error().decode()
