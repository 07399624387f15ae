"""GPU tests of the strand model rendered from its polylines (renderer.render_hair_strands: gh_strand_midpoints, the
strand instantiation of the projection kernels, gh_strand_backward):

* the kernels against PyTorch autograd of the restated strand geometry + projection (tests/_strands.py, pinned on the
  reference's GaussianModelCurves by tests/test_strands_cpu.py) with a trainable camera, at the stage-3 size and at
  strand lengths around the warp width, in both incoming-gradient modes (API tensors, the blend backward's records);
* the strand-mode binned forward bit for bit against the two-kernel path;
* render_hair_strands against the reference's own initialize_gaussians_hair() + render_hair() running on the
  reference's own rasterizer build: everything a trainer reads back;
* the NaN guard with FusedAdam over the four strand parameter groups, and the API's errors."""
import os
import sys
import types

import pytest
import torch

import _util
from _util import rel_err

sys.path.insert(0, os.path.join(_util.ROOT, "oracle"))
sys.path.insert(0, os.path.join(_util.ROOT, "tests"))
import _strands  # noqa: E402
import ref_python  # noqa: E402

pytestmark = pytest.mark.gpu
REL_TOL = 1e-4
synth = _util.synth


def _trainable_camera(cam, dev):
    camg = dict(cam)
    for k in ("world_view_transform", "full_proj_transform", "camera_center"):
        camg[k] = cam[k].to(dev).requires_grad_(True)
    camg["tanfovx"] = torch.tensor(cam["tanfovx"], dtype=torch.float32, device=dev, requires_grad=True)
    camg["tanfovy"] = torch.tensor(cam["tanfovy"], dtype=torch.float32, device=dev, requires_grad=True)
    return camg


def _pack(poly_dev, xyz, cam, W, H, deg=3):
    from gaussianhaircut_b200 import projection
    return projection.pack_inputs(xyz, poly_dev["scale"], None, poly_dev["dirs"].reshape(-1, 3), poly_dev["f_dc"],
                                  poly_dev["f_rest"], None, None, poly_dev["conf"], cam["world_view_transform"],
                                  cam["full_proj_transform"], cam["camera_center"], cam["tanfovx"], cam["tanfovy"], W, H, deg,
                                  1.0, projection.HAIR_STRANDS)


@pytest.mark.parametrize("S,L,W,H,mode", [(30000, 99, 1920, 1080, "tensors"), (30000, 99, 1920, 1080, "records"),
                                          (400, 1, 250, 187, "tensors"), (400, 31, 250, 187, "records"),
                                          (400, 32, 250, 187, "tensors"), (400, 33, 250, 187, "records"),
                                          (60, 257, 250, 187, "tensors"), (60, 257, 250, 187, "records")])
def test_strand_kernels_match_autograd(cuda_device, S, L, W, H, mode):
    from gaussianhaircut_b200 import projection, _C
    dev = cuda_device
    poly = _strands.make_strand_polylines(S, L, seed=7)
    cam = synth.make_camera(13, W, H)
    camg = _trainable_camera(cam, dev)
    leaves = {k: poly[k].to(dev).requires_grad_(True) for k in ("dirs", "f_dc", "f_rest", "conf")}
    origins = poly["origins"].to(dev)
    scale = torch.full((1,), poly["scale"], device=dev)
    ref, geo = _strands.project_strands_reference(origins, leaves["dirs"], scale, leaves["f_dc"], leaves["f_rest"],
                                                  leaves["conf"], camg)
    P = S * L
    xyz = torch.empty(P, 3, device=dev)
    projection.strand_midpoints(origins, leaves["dirs"], out=xyz)
    pd = dict(leaves, scale=scale)
    pi = _pack(pd, xyz, camg, W, H)
    out = projection.project_forward(pi, want_cov3D=True)
    torch.cuda.synchronize()
    assert torch.equal(xyz, geo["xyz"].detach())          # bit-identical to torch.cumsum + the reference's midpoints
    vis = out["visible"].bool()
    flips = int((vis != ref["mask"]).sum())
    assert flips <= max(2, P // 100000), f"{flips} prefilter decisions differ"
    both = vis & ref["mask"]
    assert rel_err(out["means2D"], ref["means2D"]) <= 1e-5
    assert rel_err(out["conic"][both], ref["conic"][both]) <= REL_TOL
    assert rel_err(out["colors"], ref["colors"]) <= 1e-5
    assert rel_err(out["cov3D"], ref["cov3D"]) <= 1e-5
    assert float(out["opacity"].min()) == 1.0 and float(out["opacity"].max()) == 1.0

    m = vis[:, None].float()
    if mode == "tensors":
        g = torch.Generator().manual_seed(3)
        gin = {"means2D": torch.randn(P, 3, generator=g).to(dev), "conic": (torch.randn(P, 3, generator=g) * 1e-3).to(dev),
               "colors": torch.randn(P, 10, generator=g).to(dev)}
        gin["means2D"][:, 2] = 0.0
        conic4 = torch.zeros(P, 2, 2, device=dev)
        conic4[:, 0, 0] = gin["conic"][:, 0]; conic4[:, 0, 1] = 0.5 * gin["conic"][:, 1]; conic4[:, 1, 1] = gin["conic"][:, 2]
        d = projection.project_backward(pi, out["visible"], dL_dmeans2D=gin["means2D"], dL_dconic4=conic4, dL_dcolors=gin["colors"],
                                        dL_dopacity=torch.zeros(P, 1, device=dev), camera_grads=True, want_means2D_grad=True)
    else:
        # the blend backward's accumulation records (what render_hair_strands uses without a head block); the same
        # image gradient through the two-kernel rasterizer gives the API-shaped tensors that drive autograd
        bg = torch.tensor(synth.BG_DEFAULT, device=dev)
        empty = torch.empty(0)
        dL = synth.upstream_gradient(W, H, 4).to(dev)
        b, radii, geom, img, R, max_len = projection.project_forward_binned(pi)
        _color, binning = _C.forward_render(bg, b["colors"], radii, geom, img, R, max_len, H, W)
        _C.rasterize_gaussians_backward_records(bg, pi.xyz, radii, b["colors"], b["conic"], pi.V, pi.Pm, pi.tanx, pi.tany, dL,
                                                pi.campos, geom, R, binning, img, False)
        d = projection.project_backward(pi, b["visible"], geom_buffer=geom, camera_grads=True, want_means2D_grad=True)
        a = projection.project_forward(pi)
        R2, _c2, radii2, geom2, bin2, img2 = _C.rasterize_gaussians(
            bg, pi.xyz, empty, a["colors"], a["opacity"], empty, empty, 1.0, empty, a["conic"], pi.V, pi.Pm, pi.tanx, pi.tany,
            H, W, empty, 3, pi.campos, False, False)
        g9 = _C.rasterize_gaussians_backward(bg, pi.xyz, radii2, a["colors"], empty, empty, 1.0, empty, a["conic"], pi.V, pi.Pm,
                                             pi.tanx, pi.tany, dL, empty, 3, pi.campos, geom2, R2, bin2, img2, False)
        gc = g9[5].reshape(P, 4)
        gin = {"means2D": g9[0].clone(), "colors": g9[1], "conic": torch.stack([gc[:, 0], 2.0 * gc[:, 1], gc[:, 3]], dim=-1)}
        gin["means2D"][:, 2] = 0.0
    projection.strand_backward(S, L, d["xyz"], d["dirs"])
    torch.cuda.synchronize()
    assert d["scaling"] is None and d["rotation"] is None
    sum((ref[k] * gin[k] * m).sum() for k in gin).backward()
    for k, src in (("dirs", "dirs"), ("f_dc", "f_dc"), ("f_rest", "f_rest"), ("conf", "conf")):
        gref = leaves[src].grad
        e = rel_err(d[k].reshape(gref.shape), gref)
        assert e <= REL_TOL, f"{k}: {e}"
    assert rel_err(d["viewmatrix"], camg["world_view_transform"].grad) <= REL_TOL
    assert rel_err(d["projmatrix"], camg["full_proj_transform"].grad) <= REL_TOL
    assert rel_err(d["campos"], camg["camera_center"].grad) <= REL_TOL
    assert rel_err(d["tanfov"], torch.stack([camg["tanfovx"].grad, camg["tanfovy"].grad])) <= REL_TOL


def test_strand_binned_projection_is_bit_identical_to_the_two_kernel_path(cuda_device):
    from gaussianhaircut_b200 import projection, _C
    dev = cuda_device
    S, L, W, H = 5000, 99, 1920, 1080
    poly = _strands.make_strand_polylines(S, L, seed=4)
    cam = {k: (v.to(dev) if isinstance(v, torch.Tensor) else v) for k, v in synth.make_camera(3, W, H).items()}
    pd = {k: (v.to(dev) if isinstance(v, torch.Tensor) else v) for k, v in poly.items()}
    pd["scale"] = torch.full((1,), poly["scale"], device=dev)
    xyz = torch.empty(S * L, 3, device=dev)
    projection.strand_midpoints(pd["origins"], pd["dirs"], out=xyz)
    pi = _pack(pd, xyz, cam, W, H)
    bg = torch.tensor(synth.BG_DEFAULT, device=dev)
    empty = torch.empty(0)
    a = projection.project_forward(pi)
    Ra, color_a, radii_a, geom_a, bin_a, img_a = _C.rasterize_gaussians(
        bg, pi.xyz, empty, a["colors"], a["opacity"], empty, empty, 1.0, empty, a["conic"], pi.V, pi.Pm, cam["tanfovx"], cam["tanfovy"],
        H, W, empty, 3, pi.campos, False, False)
    b, radii_b, geom_b, img_b, Rb, max_len = projection.project_forward_binned(pi)
    color_b, bin_b = _C.forward_render(bg, b["colors"], radii_b, geom_b, img_b, Rb, max_len, H, W)
    torch.cuda.synchronize()
    assert Ra == Rb and Ra > 0
    for k in ("means2D", "colors", "opacity", "conic", "visible"):
        assert torch.equal(a[k], b[k]), k
    assert torch.equal(radii_a, radii_b)
    assert torch.equal(color_a, color_b)
    assert torch.equal(bin_a[:8 * Ra], bin_b[:8 * Rb])


def _weights(H, W, device, seed):
    g = torch.Generator().manual_seed(seed)
    return {k: torch.rand(c, H, W, generator=g).to(device) for k, c in (("render", 3), ("mask", 2), ("orient_angle", 1), ("orient_conf", 1))}


def _loss(pkg, Wt):
    return sum((pkg[k] * Wt[k]).sum() for k in Wt)


@pytest.mark.parametrize("S,L,n_head,W,H", [(300, 99, 20000, 512, 512), (1000, 33, 0, 250, 187), (30000, 99, 200000, 1920, 1080)],
                         ids=["300x99+head-512", "1000x33-hair-only", "30000x99+head-1080p"])
def test_render_hair_strands_matches_the_reference_pipeline(cuda_device, S, L, n_head, W, H):
    """renderer.render_hair_strands against the reference's own GaussianModelCurves.initialize_gaussians_hair() and
    render_hair() on the reference's rasterizer: maps, visibility, radii and every gradient a trainer reads."""
    if not ref_python.available() or not _util.ref_available():
        pytest.skip("reference Python sources / oracle/_ref not staged")
    from gaussianhaircut_b200 import renderer
    head = synth.make_blob_scene(n_head, seed=2, spread=0.08, max_scale=0.004) if n_head else _strands.empty_head_scene()
    poly = _strands.make_strand_polylines(S, L, seed=4)
    cam_d = synth.make_camera(7, W, H)
    bg = torch.tensor(synth.BG_DEFAULT, device=cuda_device)
    Wt = _weights(H, W, cuda_device, 9)
    ref_mod = ref_python.load_renderer("ref")
    res = {}
    for which in ("mine", "ref"):
        pc, pc_hair = _strands.make_curves_models(head, poly, cuda_device)
        cam = ref_python.make_camera(cam_d, cuda_device, trainable=True)
        if which == "mine":
            pkg = renderer.render_hair_strands(cam, pc, pc_hair, ref_python.pipe(), bg)
        else:
            pc_hair.initialize_gaussians_hair()
            pkg = ref_mod.render_hair(cam, pc, pc_hair, ref_python.pipe(), bg)
        _loss(pkg, Wt).backward()
        torch.cuda.synchronize()
        res[which] = (pkg, pc_hair, cam)
    (pa, ha, ca), (pb, hb, cb) = res["mine"], res["ref"]
    P = pb["visibility_filter"].numel()
    assert pa["visibility_filter"].numel() == P
    assert int((pa["visibility_filter"] != pb["visibility_filter"]).sum()) <= max(2, P // 100000)
    assert int((pa["radii"] != pb["radii"]).sum()) <= max(4, P // 20000)
    for k in ("render", "mask", "orient_conf"):
        assert rel_err(pa[k], pb[k]) <= REL_TOL, f"{k}: {rel_err(pa[k], pb[k])}"
    assert rel_err(pa["orient_angle"], pb["orient_angle"]) <= 1e-3
    for name in _strands.CURVES_PARAMS:
        ga, gb = getattr(ha, name).grad, getattr(hb, name).grad
        assert ga is not None and gb is not None, name
        assert ga.shape == gb.shape, name
        assert rel_err(ga, gb) <= 2 * REL_TOL, f"{name}: {rel_err(ga, gb)}"
    for name in ("world_view_transform", "full_proj_transform", "camera_center"):
        assert rel_err(getattr(ca, name).grad, getattr(cb, name).grad) <= 2 * REL_TOL, name
    assert rel_err(pa["viewspace_points"].grad, pb["viewspace_points"].grad) <= 2 * REL_TOL


def _strand_model(dev, S=40, L=33, seed=6):
    poly = _strands.make_strand_polylines(S, L, seed)
    hair = types.SimpleNamespace(active_sh_degree=3, max_sh_degree=3, pts_origins=poly["origins"].to(dev),
                                 scale=poly["scale"] * torch.ones(1, device=dev))
    for n, k in (("_dirs", "dirs"), ("_features_dc", "f_dc"), ("_features_rest", "f_rest"), ("_orient_conf", "conf")):
        setattr(hair, n, torch.nn.Parameter(poly[k].to(dev).contiguous()))
    return hair


def test_nan_guard_rides_on_the_strand_backward(cuda_device):
    """set_nan_flag with render_hair_strands: a NaN in the gradients raises the device flag and FusedAdam skips the
    step over the four strand parameter groups."""
    from gaussianhaircut_b200 import renderer
    from gaussianhaircut_b200.optim import FusedAdam
    hair = _strand_model(cuda_device)
    cam = ref_python.make_camera(synth.make_camera(3, 160, 96), cuda_device)
    bg = torch.tensor(synth.BG_DEFAULT, device=cuda_device)
    names = _strands.CURVES_PARAMS
    opt = FusedAdam([{"params": [getattr(hair, n)], "lr": 1e-5, "name": n} for n in names], eps=1e-15)
    flag = torch.zeros(1, dtype=torch.int32, device=cuda_device)
    renderer.set_nan_flag(flag)
    try:
        for poisoned in (False, True, False):
            before = hair._dirs.detach().clone()
            pkg = renderer.render_hair_strands(cam, None, hair, types.SimpleNamespace(debug=False), bg)
            g = torch.rand_like(pkg["render"])
            if poisoned:
                g[:, 40:60, 60:100] = float("nan")
            (pkg["render"] * g).sum().backward()
            assert bool(flag.item() != 0) == poisoned
            opt.step(nan_flag_in=flag)
            opt.zero_grad()
            torch.cuda.synchronize()
            assert int(flag.item()) == 0
            assert torch.equal(before, hair._dirs.detach()) == poisoned, "a poisoned step must leave the parameters untouched"
        assert opt.step_count == 2
    finally:
        renderer.set_nan_flag(None)


def test_render_hair_strands_api_errors(cuda_device):
    from gaussianhaircut_b200 import projection, renderer
    cam = ref_python.make_camera(synth.make_camera(3, 64, 48), cuda_device)
    bg = torch.tensor(synth.BG_DEFAULT, device=cuda_device)
    pipe = types.SimpleNamespace(debug=False)
    hair = _strand_model(cuda_device, S=3, L=5)
    bad = _strand_model(cuda_device, S=3, L=5)
    bad._features_dc = torch.nn.Parameter(bad._features_dc.detach()[:-1])
    with pytest.raises(RuntimeError, match="S\\*L"):
        renderer.render_hair_strands(cam, None, bad, pipe, bg)
    cpu = _strand_model("cpu", S=3, L=5)
    with pytest.raises(RuntimeError, match="no CPU path"):
        renderer.render_hair_strands(ref_python.make_camera(synth.make_camera(3, 64, 48), "cpu"), None, cpu, pipe, bg.cpu())
    arena = torch.zeros(projection.grad_arena_floats(15, with_dirs=True), device=cuda_device)
    projection.set_gradient_arena(arena)
    try:
        with pytest.raises(RuntimeError, match="arena"):
            renderer.render_hair_strands(cam, None, hair, pipe, bg)
    finally:
        projection.set_gradient_arena(None)
    # the thickness as a (1,) device tensor (what create_from_pcd stores) or as a Python float: the same render
    a = renderer.render_hair_strands(cam, None, hair, pipe, bg)["raw"]
    hair_f = _strand_model(cuda_device, S=3, L=5)
    hair_f.scale = float(hair.scale.item())
    b = renderer.render_hair_strands(cam, None, hair_f, pipe, bg)["raw"]
    assert torch.equal(a, b)


def test_strand_backward_flags_nan_totals_of_finite_direct_terms(cuda_device):
    """gh_strand_backward's own NaN check: +inf and -inf midpoint gradients on two segments of one strand give NaN
    suffix totals although every direct term is finite (the projection backward's flag would not see this)."""
    from gaussianhaircut_b200 import projection
    dev = cuda_device
    S, L = 5, 70
    d_xyz = torch.randn(S * L, 3, generator=torch.Generator().manual_seed(1)).to(dev)
    flag = torch.zeros(1, dtype=torch.int32, device=dev)
    d_dirs = torch.randn(S * L, 3, device=dev)
    projection.strand_backward(S, L, d_xyz, d_dirs, nan_flag=flag)
    torch.cuda.synchronize()
    assert int(flag.item()) == 0 and bool(torch.isfinite(d_dirs).all())
    d_xyz[2 * L + 10, 1] = float("inf")
    d_xyz[2 * L + 50, 1] = float("-inf")                # strand 2, segments 10 and 50 (second chunk of 32)
    d_dirs = torch.randn(S * L, 3, device=dev)
    projection.strand_backward(S, L, d_xyz, d_dirs, nan_flag=flag)
    torch.cuda.synchronize()
    assert int(flag.item()) == 1
    g = d_dirs.view(S, L, 3)
    assert bool(torch.isnan(g[2, :11, 1]).all())        # segments 0..10 sum both infinities
    assert bool(torch.isfinite(g[[0, 1, 3, 4]]).all())
