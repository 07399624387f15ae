"""GPU tests of the trainable cameras (cameras.CameraRig / CameraAdam, gh_camera_* kernels, DESIGN §17):

  * reference parity: the reference's own `scene.cameras.Camera` (imported unmodified, trainable_cameras =
    trainable_intrinsics = use_barf = True, random residuals) against the rig: the four outputs, and the 8 gradients
    for random upstream gradients against autograd through the Camera properties;
  * training parity: the reference's camera loop (Camera, torch.optim.Adam(eps=1e-15), its translation schedule) around
    renderer.render against the rig with CameraAdam, 12 iterations over 8 views; only visited cameras move;
  * captured equals eager: CapturedTrainStep with trainable cameras against the eager loop, bit for bit under
    torch.use_deterministic_algorithms, across a forced binning overflow, a train_cameras switch and a
    densify_and_prune between steps;
  * render_hair / render_hair_strands with rig views (trainable and frozen) against the same renderers with the
    reference's own Camera: maps, `_dirs.grad` and the camera gradients;
  * guards: a NaN camera gradient skips only the camera step; an out-of-range device index sets
    GH_STATUS_CAMERA_INDEX and leaves every table unchanged.
"""
import importlib.util
import os
import sys
import types

import numpy as np
import pytest
import torch

import _util

sys.path.insert(0, os.path.join(_util.ROOT, "oracle"))
import ref_python  # noqa: E402
import synth  # noqa: E402

pytestmark = pytest.mark.gpu

NAMES = ("_xyz", "_features_dc", "_features_rest", "_opacity", "_label", "_scaling", "_rotation", "_orient_conf")
KEYS = ("xyz", "f_dc", "f_rest", "opacity", "label", "scaling", "rotation", "conf")
GNAMES = ("xyz", "f_dc", "f_rest", "opacity", "label", "scaling", "rotation", "orient_conf")
LRS = (1.6e-4, 2.5e-3, 2.5e-4, 5e-2, 2.5e-3, 5e-3, 1e-3, 1e-3)
LAMBDAS = (0.8, 0.2, 0.1, 0.1)
CAM_LRS = (1e-3, 1e-3, 1e-3)           # cam_rotation_lr, cam_translation_lr_init, cam_fov_lr (arguments/__init__.py)


@pytest.fixture
def det():
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(prev, warn_only=warn)


def _ref_camera_module():
    src = ref_python.ref_src_dir()
    if src is None or not os.path.isfile(os.path.join(src, "scene", "cameras.py")):
        pytest.skip("the reference's Python sources are not available")
    ref_python.install_stubs()
    if src not in sys.path:
        sys.path.insert(0, src)
    name = "gh_ref_scene_cameras"
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, os.path.join(src, "scene", "cameras.py"))
        mod = importlib.util.module_from_spec(spec)
        sys.modules[name] = mod
        spec.loader.exec_module(mod)
    return sys.modules[name]


def _ref_cameras(n, W, H, seed=0, residuals=True):
    """n reference Cameras on the synthetic ring, trainable (BARF + intrinsics), with random residuals."""
    Camera = _ref_camera_module().Camera
    gen = torch.Generator().manual_seed(seed)
    cams = []
    for k in range(n):
        d = synth.make_camera(8 * k, W, H, focal_factor=1.0 + 0.1 * k)
        w2c = d["world_view_transform"].double().T.numpy()
        R, T = w2c[:3, :3].T.copy(), w2c[:3, 3].copy()
        z1, z3 = torch.zeros(1, H, W), torch.zeros(3, H, W)
        cam = Camera(k, R, T, float(d["FoVx"]), float(d["FoVy"]), W, H, z3, z1, z1, z1, z1, z1, f"view_{k:02d}", k,
                     trainable_cameras=True, use_barf=True, trainable_intrinsics=True)
        if residuals:
            with torch.no_grad():
                ang = [0.0, 1e-6, 0.01, 0.05, 0.2, 0.02, 0.1, 0.003][k % 8]
                w = torch.randn(3, generator=gen)
                cam._rotation_res.copy_(w / w.norm() * ang)
                cam._translation_res.copy_(torch.randn(3, generator=gen) * 0.02)
                cam._fov_res.copy_((torch.rand(2, generator=gen) - 0.5) * 0.4)
        cams.append(cam)
    return cams


def _rel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30))


def test_rig_matches_reference_camera(cuda_device):
    from gaussianhaircut_b200.cameras import CameraRig
    cams = _ref_cameras(8, 640, 480)
    rig = CameraRig.from_cameras(cams)
    gen = torch.Generator().manual_seed(5)
    worst_f, worst_b = 0.0, 0.0
    for i, cam in enumerate(cams):
        view = rig.view(i)
        ref = (cam.world_view_transform, cam.full_proj_transform, cam.camera_center,
               torch.stack([torch.tan(cam.FoVx * 0.5).reshape(()), torch.tan(cam.FoVy * 0.5).reshape(())]))
        mine = (view.world_view_transform, view.full_proj_transform, view.camera_center, view.tan_fov)
        for a, b in zip(mine, ref):
            worst_f = max(worst_f, _rel(a.detach(), b.detach()))
        g = [torch.randn(t.shape, generator=gen).to(cuda_device) for t in ref]
        loss_ref = sum((a * b).sum() for a, b in zip(ref, g))
        loss_ref.backward()
        loss_mine = sum((a * b).sum() for a, b in zip(mine, g))
        loss_mine.backward()
        want = torch.cat([cam._rotation_res.grad, cam._translation_res.grad, cam._fov_res.grad])
        got = rig.grad[i]
        assert int(rig.touched[i]) == 1
        worst_b = max(worst_b, _rel(got, want))
    print(f"camera parity: worst forward rel err {worst_f:.3e}, worst gradient rel err {worst_b:.3e}")
    # the reference's float32 chain (series, matmuls, torch.inverse) and its float32 autograd against this
    # repository's rounding and its double backward.  Measured on an H100: 1.1e-7 forward, 2.2e-7 gradients; the
    # bounds leave about 10x of that
    assert worst_f <= 1e-6
    assert worst_b <= 2e-6
    assert rig.residuals.grad is None


def _model(dev, strands):
    from gaussianhaircut_b200.optim import FusedAdam
    raw = synth.raw_params_from_scene(synth.make_strand_scene(strands, seed=0), "gaussian_model")
    pc = types.SimpleNamespace(active_sh_degree=3, max_sh_degree=3, percent_dense=0.01)
    for n, k in zip(NAMES, KEYS):
        setattr(pc, n, torch.nn.Parameter(raw[k].to(dev).contiguous()))
    pc.optimizer = FusedAdam([{"params": [getattr(pc, n)], "lr": lr, "name": g} for n, g, lr in zip(NAMES, GNAMES, LRS)],
                             eps=1e-15, capturable=True)
    P = pc._xyz.shape[0]
    pc.xyz_gradient_accum = torch.zeros(P, 1, device=dev)
    pc.denom = torch.zeros(P, 1, device=dev)
    pc.max_radii2D = torch.zeros(P, device=dev)
    return pc


def _gts(dev, W, H, n=3):
    gen = torch.Generator().manual_seed(11)
    return [(torch.rand(3, H, W, generator=gen).to(dev), (torch.rand(2, H, W, generator=gen) > 0.3).float().to(dev),
             torch.rand(1, H, W, generator=gen).to(dev), torch.rand(1, H, W, generator=gen).to(dev)) for _ in range(n)]


def _translation_schedule():
    """The reference's own translation schedule (utils/general_utils.py get_expon_lr_func, called as
    train_gaussians.py:61-63 calls it), over a short run so that the rate changes every iteration."""
    _ref_camera_module()                      # puts the reference's sources on sys.path
    from utils.general_utils import get_expon_lr_func
    return get_expon_lr_func(lr_init=CAM_LRS[1], lr_final=CAM_LRS[1] * 0.01, max_steps=30)


def _render_step(pc, cam, gt, bg, ws):
    from gaussianhaircut_b200 import renderer, losses as ghl
    renders, _radii, _vs = renderer.render_raw(cam, pc, types.SimpleNamespace(debug=False), bg)
    l8, dL = ghl.image_loss_forward_backward(renders.detach(), *gt, *LAMBDAS, workspace=ws)
    renders.backward(dL)
    pc.optimizer.step()
    pc.optimizer.zero_grad(set_to_none=True)
    return l8


def test_training_parity_with_reference_loop(cuda_device):
    from gaussianhaircut_b200 import losses as ghl
    from gaussianhaircut_b200.cameras import CameraAdam, CameraRig
    W, H = 512, 384
    cams = _ref_cameras(10, W, H, residuals=False)
    rig = CameraRig.from_cameras(cams)
    ref_opt = torch.optim.Adam([{"params": [c._rotation_res for c in cams], "lr": CAM_LRS[0], "name": "rotation"},
                                {"params": [c._translation_res for c in cams], "lr": CAM_LRS[1], "name": "translation"},
                                {"params": [c._fov_res for c in cams], "lr": CAM_LRS[2], "name": "fov"}], lr=0.0, eps=1e-15)
    cam_opt = CameraAdam(rig, *CAM_LRS)
    pa, pb = _model(cuda_device, 300), _model(cuda_device, 300)
    bg = torch.tensor(synth.BG_DEFAULT, device=cuda_device)
    ws = torch.empty(ghl.workspace_elems(W, H), dtype=torch.float64, device=cuda_device)
    gts = _gts(cuda_device, W, H)
    order = [0, 1, 2, 3, 4, 5, 6, 7, 0, 3, 0, 5]          # 8 of the 10 views; views 8 and 9 are never visited
    schedule = _translation_schedule()
    for it, k in enumerate(order):
        for opt in (ref_opt, cam_opt):
            for g in opt.param_groups:
                if g["name"] == "translation":
                    g["lr"] = schedule(it)
        _render_step(pa, cams[k], gts[it % 3], bg, ws)
        ref_opt.step()
        ref_opt.zero_grad()
        _render_step(pb, rig.view(k), gts[it % 3], bg, ws)
        cam_opt.step()
        cam_opt.zero_grad()
    torch.cuda.synchronize()
    ref_rows = torch.stack([torch.cat([c._rotation_res, c._translation_res, c._fov_res]).detach() for c in cams])
    # Adam normalises every update to about one learning rate, so a camera gradient near zero whose float32 autograd
    # value (reference) and double value (here) differ moves its residual differently: bound the difference by a
    # fraction of one step
    d_cam = float((rig.residuals.detach() - ref_rows).abs().max())
    d_gauss = max(_util.rel_err(getattr(pb, n).detach(), getattr(pa, n).detach()) for n in NAMES)
    print(f"training parity: residuals {d_cam:.3e} (learning rate {CAM_LRS[0]:.0e}), Gaussians rel {d_gauss:.3e}")
    assert d_cam <= 0.05 * min(CAM_LRS)
    assert d_gauss <= 1e-3
    steps = [order.count(k) for k in range(10)]
    assert cam_opt.steps.tolist() == steps
    assert torch.count_nonzero(rig.residuals.detach()[8:]) == 0
    assert all(int(ref_opt.state[cams[k]._rotation_res]["step"]) == steps[k] for k in range(8))


class _CamPair:
    """An eager model + rig and a captured one from the same initialisation, stepped on the same inputs."""

    def __init__(self, dev, strands, W, H, capacity=None):
        from gaussianhaircut_b200 import losses as ghl
        from gaussianhaircut_b200.cameras import CameraAdam, CameraRig
        from gaussianhaircut_b200.graphs import CapturedTrainStep
        cams = _ref_cameras(8, W, H)
        self.W, self.H = W, H
        self.eager, self.capt = _model(dev, strands), _model(dev, strands)
        self.rig_e, self.rig_c = CameraRig.from_cameras(cams), CameraRig.from_cameras(cams)
        self.opt_e = CameraAdam(self.rig_e, *CAM_LRS)
        self.opt_c = CameraAdam(self.rig_c, *CAM_LRS, capturable=True)
        self.bg = torch.tensor(synth.BG_DEFAULT, device=dev)
        self.ws = torch.empty(ghl.workspace_elems(W, H), dtype=torch.float64, device=dev)
        self.nan = torch.zeros(1, dtype=torch.int32, device=dev)
        self.step = CapturedTrainStep(self.capt, self.capt.optimizer, W, H, self.bg, LAMBDAS, capacity=capacity,
                                      cameras=self.rig_c, camera_optimizer=self.opt_c)
        self.schedule = _translation_schedule()

    def run(self, it, k, gt, train=True):
        from gaussianhaircut_b200 import renderer, losses as ghl, densify
        for opt in (self.opt_e, self.opt_c):
            opt.param_groups[1]["lr"] = self.schedule(it)
        for pc in (self.eager, self.capt):
            for g, lr in zip(pc.optimizer.param_groups, LRS):
                g["lr"] = lr * (0.97 ** it)
        pc = self.eager
        renderer.set_nan_flag(self.nan)
        try:
            renders, radii, viewspace = renderer.render_raw(self.rig_e.view(k, requires_grad=train), pc,
                                                            types.SimpleNamespace(debug=False), self.bg)
            le, dL = ghl.image_loss_forward_backward(renders.detach(), *gt, *LAMBDAS, workspace=self.ws)
            renders.backward(dL)
            with torch.no_grad():
                densify.update_max_radii(pc, radii)
                densify.add_densification_stats(pc, viewspace, radii > 0)
            pc.optimizer.step(nan_flag_in=self.nan)
            pc.optimizer.zero_grad(set_to_none=True)
            if train:
                self.opt_e.step()
        finally:
            renderer.set_nan_flag(None)
        lc = self.step.step(self.rig_c.view(k), *gt, train_cameras=train)
        torch.cuda.synchronize()
        assert torch.equal(le.cpu(), lc), f"iteration {it}: losses"
        for n in NAMES:
            a, b = getattr(self.eager, n), getattr(self.capt, n)
            assert torch.equal(a, b), f"iteration {it}: {n}"
            for m in ("exp_avg", "exp_avg_sq"):
                assert torch.equal(self.eager.optimizer.state[a][m], self.capt.optimizer.state[b][m]), f"iteration {it}: {n}.{m}"
        for n in ("xyz_gradient_accum", "denom", "max_radii2D"):
            assert torch.equal(getattr(self.eager, n), getattr(self.capt, n)), f"iteration {it}: {n}"
        assert torch.equal(self.eager.optimizer.step_state, self.capt.optimizer.step_state)
        assert torch.equal(self.rig_e.residuals, self.rig_c.residuals), f"iteration {it}: residuals"
        for n in ("exp_avg", "exp_avg_sq", "steps"):
            assert torch.equal(getattr(self.opt_e, n), getattr(self.opt_c, n)), f"iteration {it}: camera {n}"
        assert torch.count_nonzero(self.rig_c.touched) == 0 and torch.count_nonzero(self.rig_c.grad) == 0


@pytest.mark.parametrize("strands, W, H", [(300, 512, 384), (5000, 1920, 1080)])
def test_captured_equals_eager_with_cameras(cuda_device, det, strands, W, H):
    pair = _CamPair(cuda_device, strands, W, H)
    gts = _gts(cuda_device, W, H)
    for it in range(12):
        pair.run(it, it % 8, gts[it % 3])
    assert pair.step.replays == 12 - 2 and pair.step.captures == 1 + pair.step.overflows
    assert pair.opt_c.steps.tolist() == [2, 2, 2, 2, 1, 1, 1, 1]


def test_captured_cameras_overflow_and_train_switch(cuda_device, det, monkeypatch):
    from gaussianhaircut_b200 import graphs
    W, H = 512, 384
    pair = _CamPair(cuda_device, 300, W, H)
    gts = _gts(cuda_device, W, H)
    orig_policy = graphs.capacity_for
    monkeypatch.setattr(graphs, "capacity_for", lambda r: 64)   # the first capture is too small: its replay overflows
    for it in range(6):
        # the overflowed replay leaves every table (camera rows included) untouched and the eager rerun trains: the
        # comparison with the eager loop after every iteration would fail otherwise
        pair.run(it, it % 8, gts[it % 3])
        if pair.step.overflows:
            monkeypatch.setattr(graphs, "capacity_for", orig_policy)
    assert pair.step.overflows == 1
    captures = pair.step.captures
    for it in range(6, 12):                                     # iterations_cam reached: the cameras freeze
        pair.run(it, it % 8, gts[it % 3], train=False)
    assert pair.step.captures == captures + 1
    assert pair.opt_c.steps.tolist() == [1, 1, 1, 1, 1, 1, 0, 0]


def test_nan_gradient_skips_only_the_camera_step(cuda_device):
    from gaussianhaircut_b200.cameras import CameraAdam, CameraRig
    rig = CameraRig.from_cameras(_ref_cameras(4, 64, 48))
    opt = CameraAdam(rig, *CAM_LRS)
    before = rig.residuals.detach().clone()
    d = torch.zeros(37, device=cuda_device)
    d[0] = float("nan")
    rig.backward(rig.indices[1:2], d)
    assert int(rig.nan_flag) == 1 and int(rig.touched[1]) == 1
    opt.step()
    torch.cuda.synchronize()
    assert torch.equal(rig.residuals.detach(), before) and opt.steps.tolist() == [0, 0, 0, 0]
    assert torch.count_nonzero(opt.exp_avg) == 0 and torch.count_nonzero(opt.exp_avg_sq) == 0
    assert int(rig.nan_flag) == 0 and torch.count_nonzero(rig.touched) == 0 and torch.count_nonzero(rig.grad) == 0
    # the next finite gradient steps normally
    d[0] = 1.0
    rig.backward(rig.indices[1:2], d)
    opt.step()
    assert opt.steps.tolist() == [0, 1, 0, 0] and not torch.equal(rig.residuals.detach()[1], before[1])


def test_out_of_range_index_touches_nothing(cuda_device):
    from gaussianhaircut_b200.cameras import CameraRig, STATUS_CAMERA_INDEX
    rig = CameraRig.from_cameras(_ref_cameras(3, 64, 48))
    tables = [rig.residuals.detach(), rig.base, rig.grad, rig.touched, rig.nan_flag]
    saved = [t.clone() for t in tables]
    out = torch.full((37,), 7.0, device=cuda_device)
    for bad in (3, -1, 1 << 30):
        idx = torch.tensor([bad], dtype=torch.int32, device=cuda_device)
        rig.status.zero_()
        rig.forward(idx, out=out)
        assert int(rig.status) == STATUS_CAMERA_INDEX
        rig.status.zero_()
        rig.backward(idx, torch.ones(37, device=cuda_device))
        assert int(rig.status) == STATUS_CAMERA_INDEX
    torch.cuda.synchronize()
    assert bool((out == 7.0).all())
    for a, b in zip(tables, saved):
        assert torch.equal(a, b)


def test_captured_cameras_densify_recaptures(cuda_device, det):
    from gaussianhaircut_b200 import densify
    W, H = 512, 384
    pair = _CamPair(cuda_device, 300, W, H)
    gts = _gts(cuda_device, W, H)
    P0 = pair.eager._xyz.shape[0]
    for it in range(12):
        pair.run(it, it % 8, gts[it % 3])
        if it == 5:
            for pc in (pair.eager, pair.capt):
                torch.manual_seed(1000 + it)
                torch.cuda.manual_seed(1000 + it)
                densify.densify_and_prune(pc, 2e-5, 0.005, 0.1, None)
    assert pair.eager._xyz.shape[0] != P0, "densify_and_prune changed nothing"
    # the densification changes P and the Gaussian optimizer state: two eager warm-ups, then a second capture that
    # carries on with the same camera tables
    assert pair.step.captures == 2
    assert pair.opt_c.steps.tolist() == [2, 2, 2, 2, 1, 1, 1, 1]


def _weights(H, W, device, seed):
    g = torch.Generator().manual_seed(seed)
    return {k: torch.rand(c, H, W, generator=g).to(device) for k, c in (("render", 3), ("mask", 2), ("orient_angle", 1), ("orient_conf", 1))}


@pytest.mark.parametrize("trainable", [True, False], ids=["trainable", "frozen"])
@pytest.mark.parametrize("which", ["render_hair", "render_hair_strands"])
def test_hair_renderers_with_rig_views(cuda_device, which, trainable):
    """render_hair / render_hair_strands (head block + strands) with a rig view against the same renderer with the
    reference's own Camera: the maps, the strand gradients and, for the trainable view, the camera gradients, within
    the bounds of tests/test_gpu_strands.py (REL_TOL = 1e-4 on the maps, 2e-4 on gradients, 1e-3 on the angle)."""
    sys.path.insert(0, os.path.join(_util.ROOT, "tests"))
    import _strands
    from gaussianhaircut_b200 import renderer
    from gaussianhaircut_b200.cameras import CameraRig
    REL_TOL = 1e-4
    S, L, n_head, W, H = 300, 33, 20000, 512, 512
    head = synth.make_blob_scene(n_head, seed=2, spread=0.08, max_scale=0.004)
    poly = _strands.make_strand_polylines(S, L, seed=4)
    cams = _ref_cameras(4, W, H)
    i = 3                                                      # rotation residual 0.05 rad, FoV residuals within +-0.2
    if not trainable:
        for c in cams:
            for p in (c._rotation_res, c._translation_res, c._fov_res):
                p.requires_grad_(False)
    rig = CameraRig.from_cameras(cams)
    bg = torch.tensor(synth.BG_DEFAULT, device=cuda_device)
    Wt = _weights(H, W, cuda_device, 9)
    res = {}
    for arm in ("rig", "ref"):
        pc, pc_hair = _strands.make_curves_models(head, poly, cuda_device)
        cam = rig.view(i, requires_grad=trainable) if arm == "rig" else cams[i]
        if which == "render_hair":
            pc_hair.initialize_gaussians_hair()
            pkg = renderer.render_hair(cam, pc, pc_hair, ref_python.pipe(), bg)
        else:
            pkg = renderer.render_hair_strands(cam, pc, pc_hair, ref_python.pipe(), bg)
        sum((pkg[k] * Wt[k]).sum() for k in Wt).backward()
        torch.cuda.synchronize()
        res[arm] = (pkg, pc_hair)
    (pa, ha), (pb, hb) = res["rig"], res["ref"]
    P = pb["visibility_filter"].numel()
    assert int((pa["visibility_filter"] != pb["visibility_filter"]).sum()) <= max(2, P // 100000)
    for k in ("render", "mask", "orient_conf"):
        assert _util.rel_err(pa[k], pb[k]) <= REL_TOL, f"{k}: {_util.rel_err(pa[k], pb[k])}"
    assert _util.rel_err(pa["orient_angle"], pb["orient_angle"]) <= 1e-3
    assert ha._dirs.grad is not None and hb._dirs.grad is not None
    assert _util.rel_err(ha._dirs.grad, hb._dirs.grad) <= 2 * REL_TOL, _util.rel_err(ha._dirs.grad, hb._dirs.grad)
    c = cams[i]
    if trainable:
        want = torch.cat([c._rotation_res.grad, c._translation_res.grad, c._fov_res.grad])
        err = _util.rel_err(rig.grad[i], want)
        print(f"{which}: camera gradient rel err {err:.3e}")
        assert err <= 2 * REL_TOL
        assert rig.touched.tolist() == [0, 0, 0, 1]
    else:
        assert c._rotation_res.grad is None and torch.count_nonzero(rig.touched) == 0
        assert torch.count_nonzero(rig.grad) == 0
