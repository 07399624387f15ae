"""CPU tests: pin Oracle-B (oracle/gh_oracle.c) against

  * golden vectors produced by the REFERENCE ITSELF (its CUDA extension, built in place and run on a
    GPU by tests/golden/make_golden.py): integer/bit state exact, floats to tolerance;
  * golden vectors produced by the reference's own PYTHON restatement of stage 1
    (tests/golden/make_golden_pyref.py, run in the build container).
"""
import glob
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import oracle  # noqa: E402

GOLDEN = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "*_*.npz")))
GOLDEN = [g for g in GOLDEN if not os.path.basename(g).startswith(("pyref", "loss_"))]
LOSS_GOLDEN = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "loss_*.npz")))
GRADS = ("dL_dmeans2D", "dL_dcolors", "dL_dopacity", "dL_dmeans3D", "dL_dcov3D", "dL_dconic", "dL_dsh",
         "dL_dscales", "dL_drotations")


def _opt(d, k):
    a = d["in_" + k]
    return a if a.size else None


def _run(d):
    W, H = int(d["W"]), int(d["H"])
    kw = dict(scales=_opt(d, "scales"), rotations=_opt(d, "rotations"), cov3D_precomp=_opt(d, "cov3D_precomp"),
              conic_precomp=_opt(d, "conic_precomp"), scale_modifier=float(d["scale_modifier"]))
    fw = oracle.forward(d["in_means3D"], d["in_opacities"], d["in_colors_precomp"], d["viewmatrix"], d["projmatrix"],
                        float(d["tanfovx"]), float(d["tanfovy"]), W, H, d["bg"], **kw)
    bw = oracle.backward(fw, d["dL_dout"], d["in_means3D"], d["in_colors_precomp"], d["viewmatrix"], d["projmatrix"],
                         float(d["tanfovx"]), float(d["tanfovy"]), W, H, d["bg"], **kw)
    return fw, bw


def test_golden_present():
    assert len(GOLDEN) >= 5, "golden vectors from the reference CUDA build are missing"


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[:-4] for p in GOLDEN])
def test_oracle_matches_reference_cuda_build(path):
    d = np.load(path)
    fw, bw = _run(d)
    vis = d["radii"] > 0
    # integer / bit-level state: exact
    assert fw["num_rendered"] == int(d["R"])
    assert np.array_equal(fw["radii"], d["radii"])
    assert np.array_equal(fw["tiles_touched"][vis], d["st_tiles_touched"][vis])
    assert np.array_equal(fw["depths"].view(np.uint32)[vis], d["st_depths"].view(np.uint32)[vis])
    assert np.array_equal(fw["means2D"].view(np.uint32)[vis], d["st_means2D"].view(np.uint32)[vis])
    assert np.array_equal(fw["conic_opacity"].view(np.uint32)[vis], d["st_conic_opacity"].view(np.uint32)[vis])
    assert np.array_equal(fw["keys"], d["st_keys"]), "tile|depth keys differ"
    assert np.array_equal(fw["point_list"], d["st_point_list"]), "sorted order differs"
    assert np.array_equal(fw["ranges"], d["st_ranges"])
    assert np.array_equal(fw["n_contrib"], d["st_n_contrib"])
    # floats: the CPU exp differs from CUDA's ex2.approx-based expf by <= 2 ulp
    scale = np.abs(d["out_color"]).reshape(10, -1).max(axis=1).clip(1e-12)[:, None, None]
    assert (np.abs(fw["out_color"] - d["out_color"]) / scale).max() <= 1e-5
    assert np.abs(fw["final_T"] - d["st_final_T"]).max() <= 1e-6
    for n in GRADS:
        a, b = bw[n].astype(np.float64).ravel(), d["g_" + n].astype(np.float64).ravel()
        assert a.shape == b.shape, n
        nb = np.linalg.norm(b)
        err = 0.0 if (nb == 0 and np.linalg.norm(a) == 0) else np.linalg.norm(a - b) / max(nb, 1e-300)
        assert err <= 1e-4, f"{n}: {err}"


def test_oracle_matches_reference_python_stage1():
    """Independent pin: the authors' PyTorch restatement (float32, different operation order, quaternion
    re-normalised, det + 1e-12) -> tolerance, not bits."""
    d = np.load(os.path.join(ROOT, "tests", "golden", "pyref_stage1.npz"))
    W, H = int(d["W"]), int(d["H"])
    P = d["xyz"].shape[0]
    colors = np.zeros((P, 10), np.float32)
    op = np.ones((P, 1), np.float32)
    bg = np.zeros(10, np.float32)
    fw = oracle.forward(d["xyz"], op, colors, d["viewmatrix"], d["projmatrix"], float(d["tanfovx"]), float(d["tanfovy"]),
                        W, H, bg, scales=d["scaling"], rotations=d["rotation"])
    assert np.array_equal(fw["radii"] > 0, d["points_mask"])
    np.testing.assert_allclose(fw["cov3D"], d["cov3D"], rtol=2e-5, atol=1e-12)
    np.testing.assert_allclose(fw["conic_opacity"][:, :3], d["conic"], rtol=2e-4, atol=1e-6)
    np.testing.assert_allclose(fw["depths"], d["depths"][:, 0], rtol=1e-6)
    px = ((d["mean2d_ndc"][:, 0] + 1.0) * W - 1.0) * 0.5
    py = ((d["mean2d_ndc"][:, 1] + 1.0) * H - 1.0) * 0.5
    np.testing.assert_allclose(fw["means2D"][:, 0], px, atol=2e-4)
    np.testing.assert_allclose(fw["means2D"][:, 1], py, atol=2e-4)
    # the caller-side conic fed back as conic_precomp gives the same radii/tiles as the native path
    fw2 = oracle.forward(d["xyz"], op, colors, d["viewmatrix"], d["projmatrix"], float(d["tanfovx"]), float(d["tanfovy"]),
                         W, H, bg, scales=d["scaling"], rotations=d["rotation"], conic_precomp=d["conic"])
    assert (fw2["radii"] != fw["radii"]).mean() < 0.01


def test_synth_preamble_matches_reference_python():
    """oracle/synth.py restates the caller preamble for the bench/tests; pin it too."""
    import torch
    import synth
    d = np.load(os.path.join(ROOT, "tests", "golden", "pyref_stage1.npz"))
    scene = synth.make_strand_scene(int(d["strands"]), seed=int(d["seed"]))
    cam = synth.make_camera(int(d["cam_k"]), int(d["W"]), int(d["H"]))
    pre = synth.caller_preamble(scene, cam)
    np.testing.assert_allclose(pre["conic"].numpy(), d["conic"], rtol=2e-4, atol=1e-6)
    np.testing.assert_allclose(pre["means2D"].numpy(), d["mean2d_ndc"], rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(pre["cov3D"].numpy(), d["cov3D"], rtol=2e-5, atol=1e-12)
    np.testing.assert_allclose(pre["depths"].numpy(), d["depths"], rtol=1e-6)
    np.testing.assert_allclose(pre["colors"][:, :3].numpy(), np.clip(d["sh_rgb"] + 0.5, 0, None), rtol=1e-5, atol=1e-6)
    assert torch.equal(synth.filter_points(pre, scene, cam), torch.from_numpy(d["points_mask"]))


def test_synth_preamble_gradients_match_reference_python():
    """Groundwork for SURVEY 8f row 1 (fused projection preamble): the restated preamble's autograd gradients
    -- w.r.t. the Gaussian parameters AND the camera matrices -- against the reference's own PyTorch stage 1
    differentiated on the CPU (tests/golden/make_golden_pyref_grad.py)."""
    import torch
    import torch.nn.functional as F
    import synth
    d = np.load(os.path.join(ROOT, "tests", "golden", "pyref_stage1_grad.npz"))
    scene = synth.make_strand_scene(int(d["strands"]), seed=int(d["seed"]))
    cam = dict(synth.make_camera(int(d["cam_k"]), int(d["W"]), int(d["H"])))
    leaf = lambda t: t.clone().requires_grad_(True)   # noqa: E731
    xyz, log_s, rot = leaf(scene["xyz"]), leaf(torch.log(scene["scaling"])), leaf(scene["rotation"])
    f_dc, f_rest = leaf(scene["f_dc"]), leaf(scene["f_rest"])
    vm, pm, cc = leaf(cam["world_view_transform"]), leaf(cam["full_proj_transform"]), leaf(cam["camera_center"])
    cam.update(world_view_transform=vm, full_proj_transform=pm, camera_center=cc)
    sc = dict(scene, xyz=xyz, scaling=torch.exp(log_s), rotation=F.normalize(rot, dim=-1), f_dc=f_dc, f_rest=f_rest)
    pre = synth.caller_preamble(sc, cam)
    dirs = xyz - cc[None]
    dirs = dirs / dirs.norm(dim=1, keepdim=True)
    rgb = synth.eval_sh(3, torch.cat([f_dc, f_rest], dim=1).transpose(1, 2), dirs)
    g = torch.Generator().manual_seed(int(d["weight_seed"]))
    Wc, Wm, Wd, Wr = (torch.rand(t.shape, generator=g) for t in (pre["conic"], pre["means2D"], pre["depths"], rgb))
    loss = (pre["conic"] * Wc).sum() * 1e-3 + (pre["means2D"] * Wm).sum() + (pre["depths"] * Wd).sum() + (rgb * Wr).sum()
    loss.backward()
    assert abs(float(loss.detach()) - float(d["loss"])) <= 2e-4 * abs(float(d["loss"]))
    for name, t in (("g_xyz", xyz), ("g_log_scaling", log_s), ("g_rotation", rot), ("g_f_dc", f_dc), ("g_f_rest", f_rest),
                    ("g_viewmatrix", vm), ("g_projmatrix", pm), ("g_campos", cc)):
        ref = torch.from_numpy(d[name])
        err = (t.grad - ref).norm().item() / max(ref.norm().item(), 1e-30)
        assert err <= 5e-4, f"{name}: relative error {err}"


def test_oracle_edge_cases():
    """R == 0 -> pure background; zero-determinant conic dropped; W,H not multiples of 16."""
    rng = np.random.default_rng(0)
    P, W, H = 50, 37, 21
    xyz = rng.normal(size=(P, 3)).astype(np.float32) * 0.05
    vm = np.eye(4, dtype=np.float32); vm[3, 2] = 1.0           # translate +1 in z (row-vector convention)
    pm = vm.copy(); pm[:, 3] = vm[:, 2]                          # w = z_view
    colors = rng.random((P, 10)).astype(np.float32)
    op = np.full((P, 1), 0.7, np.float32)
    bg = np.arange(10, dtype=np.float32)
    conic = np.tile(np.array([[0.5, 0.1, 0.4]], np.float32), (P, 1))
    conic[::5] = [1.0, 1.0, 1.0]
    fw = oracle.forward(xyz, op, colors, vm, pm, 0.5, 0.5, W, H, bg, conic_precomp=conic,
                        scales=np.ones((P, 3), np.float32), rotations=np.ones((P, 4), np.float32))
    assert (fw["radii"][::5] == 0).all() and (fw["radii"][1::5] > 0).all()
    assert fw["out_color"].shape == (10, H, W)
    vm_away = vm.copy(); vm_away[3, 2] = -5.0
    fw0 = oracle.forward(xyz, op, colors, vm_away, pm, 0.5, 0.5, W, H, bg, conic_precomp=conic)
    assert fw0["num_rendered"] == 0 and fw0["culled"] == P
    assert np.array_equal(fw0["out_color"], np.broadcast_to(bg[:, None, None], (10, H, W)))
    assert np.array_equal(oracle.mark_visible(xyz, vm), np.ones(P, bool))
    assert not oracle.mark_visible(xyz, vm_away).any()


@pytest.mark.parametrize("path", LOSS_GOLDEN, ids=[os.path.basename(p)[:-4] for p in LOSS_GOLDEN])
def test_loss_oracle_matches_reference_loss_utils(path):
    """'Next' row 4: oracle/loss_oracle.py against outputs of the reference's own loss_utils
    (tests/golden/make_golden_loss.py), values and autograd gradients."""
    import torch
    import loss_oracle
    d = np.load(path)
    renders, gt_image, gt_mask, gt_angle, gt_conf = loss_oracle.synthetic_case(int(d["W"]), int(d["H"]), int(d["seed"]),
                                                                                zero_weights=bool(d["zero_weights"]))
    renders.requires_grad_(True)
    loss, parts = loss_oracle.training_loss(renders, gt_image, gt_mask, gt_angle, gt_conf, *[float(x) for x in d["lambdas"]])
    loss.backward()
    assert abs(float(loss) - float(d["loss"])) <= 1e-6 * max(1.0, abs(float(d["loss"])))
    for k in ("Ll1", "Lssim", "Lmask", "Lorient"):
        assert abs(float(parts[k]) - float(d[k])) <= 1e-6, k
    g_ref = torch.from_numpy(d["dL_drender"])
    assert (renders.grad - g_ref).norm() <= 1e-6 * g_ref.norm()


def test_loss_golden_present():
    assert len(LOSS_GOLDEN) >= 3
