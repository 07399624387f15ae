"""GPU tests of the captured training iteration (graphs.CapturedTrainStep and the capturable entry points):

  * captured equals eager: 12 iterations over 8 cameras with different fields of view and a learning rate that changes
    every step give, after every iteration, the same parameters, moments, step count, losses and densification
    statistics bit for bit as the eager loop (deterministic mode), and agree within the fast-path tolerance otherwise;
  * one graph serves a close-up camera on the long-list sort path, an ordinary one and one that sees nothing;
  * overflow: the replay skips the update and touches nothing; the binning buffer's guard bytes stay intact; the step
    reruns eagerly, recaptures with a larger capacity and the run stays bit-identical to eager;
  * a densify_and_prune between steps recaptures and stays bit-identical;
  * trainable cameras, debug mode and an installed gradient arena are refused before anything is captured.
"""
import os
import sys
import types

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


@pytest.fixture
def det():
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(prev, warn_only=warn)


def _model(dev, strands, capturable):
    from gaussianhaircut_b200.optim import FusedAdam
    raw = synth.raw_params_from_scene(synth.make_strand_scene(strands, seed=0), "gaussian_model")
    pc = types.SimpleNamespace(active_sh_degree=3, max_sh_degree=3, percent_dense=0.01)
    for n, k in zip(NAMES, KEYS):
        setattr(pc, n, torch.nn.Parameter(raw[k].to(dev).contiguous()))
    pc.optimizer = FusedAdam([{"params": [getattr(pc, n)], "lr": lr, "name": g} for n, g, lr in zip(NAMES, GNAMES, LRS)],
                             eps=1e-15, capturable=capturable)
    P = pc._xyz.shape[0]
    pc.xyz_gradient_accum = torch.zeros(P, 1, device=dev)
    pc.denom = torch.zeros(P, 1, device=dev)
    pc.max_radii2D = torch.zeros(P, device=dev)
    return pc


def _camera(k, W, H, focal=1.2, away=False, radius=0.8):
    d = synth.make_camera(k, W, H, focal_factor=focal, radius=radius)
    if away:                        # every Gaussian behind the near plane: R = 0
        wv = d["world_view_transform"].double()
        pm_t = torch.linalg.inv(wv) @ d["full_proj_transform"].double()
        wv[3, 2] -= 10.0
        d["world_view_transform"] = wv.float().contiguous()
        d["full_proj_transform"] = (wv @ pm_t).float().contiguous()
    return d


def _gts(dev, W, H, n=3):
    gen = torch.Generator().manual_seed(11)
    return [(torch.rand(3, H, W, generator=gen).to(dev), (torch.rand(2, H, W, generator=gen) > 0.3).float().to(dev),
             torch.rand(1, H, W, generator=gen).to(dev), torch.rand(1, H, W, generator=gen).to(dev)) for _ in range(n)]


def _eager_step(pc, cam, gt, bg, ws, nan_flag):
    """The iteration of tools/train_loop.py (single GPU)."""
    from gaussianhaircut_b200 import renderer, losses as ghl, densify
    renderer.set_nan_flag(nan_flag)
    try:
        renders, radii, viewspace = renderer.render_raw(cam, pc, types.SimpleNamespace(debug=False), bg)
        l8, dL = ghl.image_loss_forward_backward(renders.detach(), *gt, *LAMBDAS, workspace=ws)
        renders.backward(dL)
        with torch.no_grad():
            densify.update_max_radii(pc, radii)
            densify.add_densification_stats(pc, viewspace, radii > 0)
        pc.optimizer.step(nan_flag_in=nan_flag)
        pc.optimizer.zero_grad(set_to_none=True)
    finally:
        renderer.set_nan_flag(None)
    return l8.cpu()


def _state(pc):
    out = {"step_state": pc.optimizer.step_state.clone(), "accum": pc.xyz_gradient_accum.clone(),
           "denom": pc.denom.clone(), "max_radii": pc.max_radii2D.clone()}
    for n in NAMES:
        p = getattr(pc, n)
        st = pc.optimizer.state[p]
        out[n], out[n + ".m"], out[n + ".v"] = p.detach().clone(), st["exp_avg"].clone(), st["exp_avg_sq"].clone()
    return out


def _set_lr(pc, it):
    for g, lr in zip(pc.optimizer.param_groups, LRS):
        g["lr"] = lr * (0.97 ** it)


class _Pair:
    """An eager model and a captured one from the same initialisation, stepped on the same inputs."""

    def __init__(self, dev, strands, W, H, capacity=None):
        from gaussianhaircut_b200 import losses as ghl
        from gaussianhaircut_b200.graphs import CapturedTrainStep
        self.dev, self.W, self.H = dev, W, H
        self.eager, self.capt = _model(dev, strands, False), _model(dev, strands, True)
        self.bg = torch.tensor(synth.BG_DEFAULT, device=dev)
        self.ws = torch.empty(ghl.workspace_elems(W, H), dtype=torch.float64, device=dev)
        self.nan = torch.zeros(1, dtype=torch.int32, device=dev)
        self.step = CapturedTrainStep(self.capt, self.capt.optimizer, W, H, self.bg, LAMBDAS, capacity=capacity)

    def run(self, it, cam, gt, exact=True):
        _set_lr(self.eager, it)
        _set_lr(self.capt, it)
        le = _eager_step(self.eager, cam, gt, self.bg, self.ws, self.nan)
        lc = self.step.step(cam, *gt)
        torch.cuda.synchronize()
        a, b = _state(self.eager), _state(self.capt)
        if exact:
            assert torch.equal(le, lc), f"iteration {it}: losses {le} vs {lc}"
            for k in a:
                assert a[k].shape == b[k].shape and torch.equal(a[k], b[k]), f"iteration {it}: {k}"
        return a, b


@pytest.mark.parametrize("strands, W, H", [(300, 512, 384), (5000, 1920, 1080)])
def test_captured_equals_eager(cuda_device, det, strands, W, H):
    pair = _Pair(cuda_device, strands, W, H)
    # eight cameras, eight fields of view
    cams = [ref_python.make_camera(_camera(8 * k, W, H, focal=1.0 + 0.1 * k), cuda_device) for k in range(8)]
    gts = _gts(cuda_device, W, H)
    for it in range(12):
        pair.run(it, cams[it % 8], gts[it % 3])
    # (a view whose R outgrows the capacity seeded by the first views reruns eagerly and recaptures: still bit-identical)
    # (an overflowed replay counts as a replay; the next step recaptures without warm-up)
    assert pair.step.replays == 12 - 2 and pair.step.captures == 1 + pair.step.overflows
    assert int(pair.capt.optimizer.step_state[0]) == 12


def test_captured_fast_path_agrees(cuda_device):
    W, H = 512, 384
    pair = _Pair(cuda_device, 300, W, H)
    cams = [ref_python.make_camera(_camera(8 * k, W, H, focal=1.0 + 0.1 * k), cuda_device) for k in range(8)]
    gts = _gts(cuda_device, W, H)
    for it in range(12):
        a, b = pair.run(it, cams[it % 8], gts[it % 3], exact=False)
    assert pair.step.replays == 12 - 2
    for n in NAMES:
        assert _util.rel_err(b[n], a[n]) <= 1e-5, n


def _max_tile_len(pc, cam, W, H):
    from gaussianhaircut_b200 import projection, renderer
    pi = projection.pack_inputs(pc._xyz, pc._scaling, pc._rotation, None, pc._features_dc, pc._features_rest, pc._opacity,
                                pc._label, pc._orient_conf, cam.world_view_transform, cam.full_proj_transform,
                                cam.camera_center, renderer._tan_half(cam.FoVx), renderer._tan_half(cam.FoVy), W, H, 3, 1.0,
                                projection.GAUSSIAN_MODEL)
    _out, _radii, _g, _i, R, max_len = projection.project_forward_binned(pi)
    return R, max_len


def test_one_graph_long_lists_and_empty_frame(cuda_device, det):
    from gaussianhaircut_b200 import _C, renderer
    W, H = 512, 384
    pair = _Pair(cuda_device, 300, W, H)
    ordinary = ref_python.make_camera(_camera(0, W, H), cuda_device)
    # a camera far enough away that the whole model falls into a few tiles: lists beyond the in-kernel sort's 1792
    close = None
    for radius in (3.0, 6.0, 12.0, 24.0):
        cam = ref_python.make_camera(_camera(0, W, H, radius=radius), cuda_device)
        if _max_tile_len(pair.eager, cam, W, H)[1] > 1792:
            close = cam
            break
    assert close is not None, "no camera reaches the long-list sort path"
    empty = ref_python.make_camera(_camera(0, W, H, away=True), cuda_device)
    R_close = _max_tile_len(pair.eager, close, W, H)[0]
    assert _max_tile_len(pair.eager, ordinary, W, H)[1] <= 1792 and _max_tile_len(pair.eager, empty, W, H)[0] == 0
    pair.step.capacity = _C.capacity_for(R_close)           # no overflow: every frame replays from the first graph
    gts = _gts(cuda_device, W, H)
    order = [ordinary, ordinary, close, ordinary, empty, close, empty, ordinary]
    for it, cam in enumerate(order):
        pair.run(it, cam, gts[it % 3])
    assert pair.step.captures == 1 and pair.step.overflows == 0 and pair.step.replays == len(order) - 2
    # the capturable forward itself: image and radii equal to render_raw's for all three cameras
    pc = pair.eager
    binning = _C.binning_workspace(pair.step.capacity, cuda_device)
    status = torch.zeros(1, dtype=torch.int32, device=cuda_device)
    for cam in (ordinary, close, empty):
        img_e, radii_e, _ = renderer.render_raw(cam, pc, types.SimpleNamespace(debug=False), pair.bg)
        c = {"viewmatrix": cam.world_view_transform, "projmatrix": cam.full_proj_transform, "campos": cam.camera_center,
             "tan_fov": torch.tensor([renderer._tan_half(cam.FoVx), renderer._tan_half(cam.FoVy)], device=cuda_device)}
        img_c, radii_c, _ = renderer.render_raw_capturable(c, pc, pair.bg, W, H, binning, pair.step.capacity, status)
        assert torch.equal(img_e, img_c) and torch.equal(radii_e, radii_c)
    assert int(status) == 0


def test_overflow_skips_then_reruns(cuda_device, det, monkeypatch):
    from gaussianhaircut_b200 import graphs
    W, H = 512, 384
    pair = _Pair(cuda_device, 300, W, H)
    cams = [ref_python.make_camera(_camera(8 * k, W, H), cuda_device) for k in range(8)]
    R0 = _max_tile_len(pair.eager, cams[0], W, H)[0]
    gts = _gts(cuda_device, W, H)
    seen = {}
    orig_eager, orig_policy = pair.step._eager, graphs.capacity_for
    # the first capture gets a capacity below every view's R
    monkeypatch.setattr(graphs, "capacity_for", lambda r: R0 // 2)

    def eager_after_replay(camera, gts_):
        if pair.step.replays > 0 and "state" not in seen:
            seen["state"], seen["status"] = _state(pair.capt), int(pair.step._host[0])
            monkeypatch.setattr(graphs, "capacity_for", orig_policy)
            pair.step.capacity = orig_policy(pair.step.r_max)
        return orig_eager(camera, gts_)

    monkeypatch.setattr(pair.step, "_eager", eager_after_replay)
    it = 0
    while pair.step.replays == 0:                           # warm-ups, then the first (overflowing) replay
        before = _state(pair.capt) if it > 0 else None
        pair.run(it, cams[it % 8], gts[it % 3])
        it += 1
    assert pair.step.overflows == 1 and seen["status"] & 1 and pair.step.capacity > R0
    for k in before:
        assert torch.equal(before[k], seen["state"][k]), f"the overflowed replay changed {k}"
    for it in range(it, it + 6):
        pair.run(it, cams[it % 8], gts[it % 3])
    assert pair.step.captures == 2 + (pair.step.overflows - 1) and pair.step.replays >= 5


def test_overflow_touches_no_record_beyond_capacity(cuda_device):
    """The capturable calls on a frame whose R exceeds the capacity: status bit, guard bytes intact, background image,
    final_T = 1, n_contrib = 0, zero radii, zero records."""
    from gaussianhaircut_b200 import _C, projection, renderer
    W, H = 512, 384
    pc = _model(cuda_device, 300, False)
    cam = ref_python.make_camera(_camera(0, W, H), cuda_device)
    R = _max_tile_len(pc, cam, W, H)[0]
    cap = R // 2
    nbytes = _C.binning_workspace(cap, cuda_device).numel()
    raw = torch.full((nbytes + 65536,), 0xA5, dtype=torch.uint8, device=cuda_device)
    binning, guard = raw[:nbytes], raw[nbytes:]
    tan = torch.tensor([renderer._tan_half(cam.FoVx), renderer._tan_half(cam.FoVy)], device=cuda_device)
    status = torch.zeros(1, dtype=torch.int32, device=cuda_device)
    nr = torch.zeros(1, dtype=torch.int32, device=cuda_device)
    pi = projection.pack_inputs(pc._xyz, pc._scaling, pc._rotation, None, pc._features_dc, pc._features_rest, pc._opacity,
                                pc._label, pc._orient_conf, cam.world_view_transform, cam.full_proj_transform,
                                cam.camera_center, 0.0, 0.0, W, H, 3, 1.0, projection.GAUSSIAN_MODEL)
    out, radii, geom, img = projection.project_forward_binned_capturable(pi, tan, binning, cap, status, nr)
    bg = torch.tensor(synth.BG_DEFAULT, device=cuda_device)
    color = _C.forward_render_capturable(bg, out["colors"], geom, binning, img, cap, H, W)
    for d in (False, True):
        torch.use_deterministic_algorithms(d)
        try:
            _C.backward_records_capturable(bg, out["colors"], radii, geom, binning, img, cap,
                                           synth.upstream_gradient(W, H, 0).to(cuda_device))
            torch.cuda.synchronize()
        finally:
            torch.use_deterministic_algorithms(False)
        P = pc._xyz.shape[0]
        a = lambda n: (n + 255) // 256 * 256  # noqa: E731
        off = a(P * 32) + a(P * 4)
        assert not bool(geom[off:off + 64 * P].any()), f"records not zero (deterministic={d})"
    assert int(status) == 1 and int(nr) == R
    assert bool((guard == 0xA5).all()), "a kernel wrote beyond the binning buffer"
    assert not bool(radii.any())
    assert torch.equal(color, bg.view(-1, 1, 1).expand_as(color))
    ex = _C.debug_export(P, W, H, 0, geom, binning, img)
    assert bool((ex["final_T"] == 1).all()) and not bool(ex["n_contrib"].any())


def test_densify_recaptures(cuda_device, det):
    from gaussianhaircut_b200 import densify
    W, H = 512, 384
    pair = _Pair(cuda_device, 300, W, H)
    cams = [ref_python.make_camera(_camera(8 * k, W, H, focal=1.0 + 0.1 * k), cuda_device) for k in range(8)]
    gts = _gts(cuda_device, W, H)
    P0 = pair.eager._xyz.shape[0]
    for it in range(12):
        pair.run(it, cams[it % 8], gts[it % 3])
        if it == 5:
            for pc in (pair.eager, pair.capt):
                torch.manual_seed(1000 + it)
                torch.cuda.manual_seed(1000 + it)
                densify.densify_and_prune(pc, 2e-5, 0.005, 0.1, None)
    assert pair.eager._xyz.shape[0] != P0, "densify_and_prune changed nothing"
    assert pair.step.captures == 2


def test_rejections(cuda_device):
    from gaussianhaircut_b200 import projection
    from gaussianhaircut_b200.graphs import CapturedTrainStep
    W, H = 256, 192
    pc = _model(cuda_device, 50, True)
    bg = torch.tensor(synth.BG_DEFAULT, device=cuda_device)
    with pytest.raises(RuntimeError, match="debug"):
        CapturedTrainStep(pc, pc.optimizer, W, H, bg, LAMBDAS, pipe=types.SimpleNamespace(debug=True))
    with pytest.raises(RuntimeError, match="capturable=True"):
        CapturedTrainStep(pc, _model(cuda_device, 50, False).optimizer, W, H, bg, LAMBDAS)
    prev = projection.set_gradient_arena(torch.zeros(projection.grad_arena_floats(pc._xyz.shape[0]), device=cuda_device))
    try:
        with pytest.raises(RuntimeError, match="gradient arena"):
            CapturedTrainStep(pc, pc.optimizer, W, H, bg, LAMBDAS)
    finally:
        projection.set_gradient_arena(prev)
    step = CapturedTrainStep(pc, pc.optimizer, W, H, bg, LAMBDAS)
    cam = ref_python.make_camera(_camera(0, W, H), cuda_device, trainable=True)
    x0 = pc._xyz.detach().clone()
    with pytest.raises(RuntimeError, match="trainable cameras"):
        step.step(cam, *_gts(cuda_device, W, H, 1)[0])
    assert step.captures == 0 and step._warm == 0 and torch.equal(pc._xyz.detach(), x0)
