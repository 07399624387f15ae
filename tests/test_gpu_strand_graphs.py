"""GPU tests of the captured strand iteration (graphs.CapturedStrandStep, renderer.render_hair_strands_capturable and
the gh_hair_strands_*_capturable entry points), on the scenes of tests/_strands.py:

  * captured equals eager: 12 iterations over 8 cameras with different fields of view and a `_dirs` learning rate that
    changes every step give, after every iteration, the same parameters, moments, step count and losses bit for bit as
    the eager iteration (render_hair_strands -> strand loss -> backward -> FusedAdam), in deterministic mode, with and
    without a head block, for both settings of the loss options; the fast path agrees within a norm-relative bound;
  * one graph serves a camera on the long-list sort path, an ordinary one and one that sees nothing, and the
    capturable render equals render_hair_strands' image and radii for all three;
  * overflow: the replay changes nothing, the guard bytes past the binning buffer stay intact, and the step reruns
    eagerly, recaptures and stays bit-identical;
  * the prior's `_dirs` gradient: added like `_dirs.grad += dirs_grad`, bit-identical; a NaN in it skips the step;
  * frozen CameraRig views; the refusals (debug mode, a gradient arena, camera tensors that require grad, a
    non-capturable optimizer) before anything is captured.
"""
import os
import sys
import types

import pytest
import torch

import _util
import _strands

sys.path.insert(0, os.path.join(_util.ROOT, "oracle"))
import ref_python  # noqa: E402
import synth  # noqa: E402

pytestmark = pytest.mark.gpu

NAMES = _strands.CURVES_PARAMS        # _dirs, _features_dc, _features_rest, _orient_conf
LRS = {"_dirs": 1.6e-4, "_features_dc": 2.5e-3, "_features_rest": 2.5e-3 / 20.0, "_orient_conf": 0.05}
LAMBDAS = (0.8, 0.2, 0.2, 0.1)
PIPE = types.SimpleNamespace(debug=False)
OPTIONS = [(True, True), (False, False)]
_SCENES = {}


@pytest.fixture
def det():
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(prev, warn_only=warn)


def _scene(S, L, n_head):
    key = (S, L, n_head)
    if key not in _SCENES:
        head = (synth.make_blob_scene(n_head, seed=2, spread=0.08, max_scale=0.004) if n_head
                else _strands.empty_head_scene())
        _SCENES.clear()
        _SCENES[key] = (head, _strands.make_strand_polylines(S, L, seed=4))
    return _SCENES[key]


def _models(dev, S, L, n_head, capturable, dirs_lr=LRS["_dirs"]):
    from gaussianhaircut_b200.optim import FusedAdam
    head, poly = _scene(S, L, n_head)
    pc, hair = _strands.make_curves_models(head, poly, dev)
    lrs = dict(LRS, _dirs=dirs_lr)
    opt = FusedAdam([{"params": [getattr(hair, n)], "lr": lrs[n], "name": n} for n in NAMES], eps=1e-15,
                    capturable=capturable)
    return pc, hair, opt


def _camera(k, W, H, focal=1.2, away=False, radius=0.8):
    d = synth.make_camera(k, W, H, focal_factor=focal, radius=radius)
    if away:                        # everything behind the near plane: R = 0
        wv = d["world_view_transform"].double()
        pm_t = torch.linalg.inv(wv) @ d["full_proj_transform"].double()
        wv[3, 2] -= 10.0
        d["world_view_transform"] = wv.float().contiguous()
        d["full_proj_transform"] = (wv @ pm_t).float().contiguous()
    return d


def _cams(dev, W, H):
    return [ref_python.make_camera(_camera(8 * k, W, H, focal=1.0 + 0.1 * k), dev) for k in range(8)]


def _gts(dev, W, H, n=3):
    gen = torch.Generator().manual_seed(11)
    return [(torch.rand(3, H, W, generator=gen).to(dev), (torch.rand(2, H, W, generator=gen) > 0.3).float().to(dev),
             torch.rand(1, H, W, generator=gen).to(dev), torch.rand(1, H, W, generator=gen).to(dev)) for _ in range(n)]


def _eager_step(pc, hair, opt, cam, gt, bg, nan_flag, options, dirs_grad=None):
    """The train_strands.py iteration of tools/strand_loss_step.py's kernel arm (+ the prior gradient)."""
    from gaussianhaircut_b200 import renderer, losses as ghl
    renderer.set_nan_flag(nan_flag)
    try:
        pkg = renderer.render_hair_strands(cam, pc, hair, PIPE, bg)
        l8, dL = ghl.image_loss_forward_backward(pkg["raw"].detach(), *gt, *LAMBDAS, stage="strands",
                                                 use_gt_orient_conf=options[0], train_orient_conf=options[1])
        pkg["raw"].backward(dL)
        if dirs_grad is not None:
            hair._dirs.grad += dirs_grad
            if bool(hair._dirs.grad.isnan().any()):
                nan_flag.fill_(1)
    finally:
        renderer.set_nan_flag(None)
    opt.step(nan_flag_in=nan_flag)
    opt.zero_grad(set_to_none=True)
    return l8.cpu()


def _state(hair, opt):
    out = {"step_state": opt.step_state.clone()}
    for n in NAMES:
        p = getattr(hair, n)
        st = opt.state[p]
        out[n], out[n + ".m"], out[n + ".v"] = p.detach().clone(), st["exp_avg"].clone(), st["exp_avg_sq"].clone()
    return out


class _Pair:
    """An eager strand model and a captured one from the same initialisation, stepped on the same inputs."""

    def __init__(self, dev, S, L, n_head, W, H, options=(True, True), capacity=None, dirs_lr=LRS["_dirs"], rigs=None):
        from gaussianhaircut_b200.graphs import CapturedStrandStep
        self.dev, self.W, self.H, self.options, self.dirs_lr = dev, W, H, options, dirs_lr
        self.eager = _models(dev, S, L, n_head, False, dirs_lr)
        self.capt = _models(dev, S, L, n_head, True, dirs_lr)
        self.bg = torch.tensor(synth.BG_DEFAULT, device=dev)
        self.nan = torch.zeros(1, dtype=torch.int32, device=dev)
        pc, hair, opt = self.capt
        self.step = CapturedStrandStep(pc, hair, opt, W, H, self.bg, LAMBDAS, use_gt_orient_conf=options[0],
                                       train_orient_conf=options[1], capacity=capacity,
                                       cameras=None if rigs is None else rigs[1])

    def set_lr(self, it, schedule=True):
        for _pc, _hair, opt in (self.eager, self.capt):
            for g in opt.param_groups:
                if g["name"] == "_dirs":
                    g["lr"] = self.dirs_lr * (0.97 ** it if schedule else 1.0)

    def run(self, it, cam, gt, exact=True, cam_c=None, dirs_grad=None, schedule=True):
        self.set_lr(it, schedule)
        le = _eager_step(*self.eager, cam, gt, self.bg, self.nan, self.options, dirs_grad)
        lc = self.step.step(cam if cam_c is None else cam_c, *gt, dirs_grad=dirs_grad)
        torch.cuda.synchronize()
        a, b = _state(*self.eager[1:]), _state(*self.capt[1:])
        if exact:
            assert torch.equal(le, lc), f"iteration {it}: losses {le} vs {lc}"
            for k in a:
                assert a[k].shape == b[k].shape and torch.equal(a[k], b[k]), f"iteration {it}: {k}"
        return a, b


@pytest.mark.parametrize("options", OPTIONS, ids=["gt_conf", "unit_weights_no_conf"])
@pytest.mark.parametrize("S, L, n_head, W, H", [(300, 99, 20000, 512, 512), (1000, 33, 0, 250, 187),
                                                (30000, 99, 200000, 1920, 1080)],
                         ids=["head_512", "hair_only_250x187", "bench_1080p"])
def test_captured_equals_eager(cuda_device, det, S, L, n_head, W, H, options):
    pair = _Pair(cuda_device, S, L, n_head, W, H, options)
    cams, gts = _cams(cuda_device, W, H), _gts(cuda_device, W, H)
    for it in range(12):
        pair.run(it, cams[it % 8], gts[it % 3])
    assert pair.step.replays == 12 - 2 and pair.step.captures == 1 + pair.step.overflows
    assert int(pair.capt[2].step_state[0]) == 12


def test_captured_fast_path_agrees(cuda_device):
    W, H = 512, 512
    # `_dirs` at the end of its schedule: at 1.6e-4, Adam's eps = 1e-15 turns gradient sign noise into +-lr steps
    pair = _Pair(cuda_device, 300, 99, 20000, W, H, dirs_lr=1.6e-6)
    cams, gts = _cams(cuda_device, W, H), _gts(cuda_device, W, H)
    for it in range(12):
        a, b = pair.run(it, cams[it % 8], gts[it % 3], exact=False, schedule=False)
    assert pair.step.replays == 12 - 2
    errs = {n: _util.rel_err(b[n], a[n]) for n in NAMES}
    print("fast path, norm-relative parameter differences:", errs)
    for n, e in errs.items():
        assert e <= 5e-5, n


def _strand_max_tile_len(hair, cam, W, H):
    """(R, longest tile list) of the strand rows alone (projection.project_forward_binned on the segments)."""
    from gaussianhaircut_b200 import projection, renderer
    S, L = hair._dirs.shape[0], hair._dirs.shape[1]
    mid = torch.empty(S * L, 3, device=hair._dirs.device)
    projection.strand_midpoints(hair.pts_origins, hair._dirs, out=mid)
    pi = projection.pack_inputs(mid, hair.scale, None, hair._dirs.reshape(-1, 3), hair._features_dc, hair._features_rest,
                                None, None, hair._orient_conf, cam.world_view_transform, cam.full_proj_transform,
                                cam.camera_center, renderer._tan_half(cam.FoVx), renderer._tan_half(cam.FoVy), W, H, 3,
                                1.0, projection.HAIR_STRANDS)
    _o, _r, _g, _i, R, max_len = projection.project_forward_binned(pi)
    return R, max_len


def _eager_R(pc, hair, cam, bg, W, H):
    """R of render_hair_strands on `cam` (the value its forward records)."""
    from gaussianhaircut_b200 import _C, renderer
    pkg = renderer.render_hair_strands(cam, pc, hair, PIPE, bg)
    return _C.last_num_rendered((bg.device.index, int(pkg["radii"].shape[0]), W, H))


def _static_camera(cam, dev):
    from gaussianhaircut_b200 import renderer
    return {"viewmatrix": cam.world_view_transform, "projmatrix": cam.full_proj_transform, "campos": cam.camera_center,
            "tan_fov": torch.tensor([renderer._tan_half(cam.FoVx), renderer._tan_half(cam.FoVy)], device=dev)}


def test_one_graph_long_lists_and_empty_frame(cuda_device, det):
    from gaussianhaircut_b200 import _C, renderer
    W, H = 512, 512
    pair = _Pair(cuda_device, 300, 99, 20000, W, H)
    pc, hair, _ = pair.eager
    ordinary = ref_python.make_camera(_camera(0, W, H), cuda_device)
    close = None                  # far enough away that the model falls into a few tiles: lists beyond 1792 records
    for radius in (3.0, 6.0, 12.0, 24.0):
        cam = ref_python.make_camera(_camera(0, W, H, radius=radius), cuda_device)
        if _strand_max_tile_len(hair, cam, W, H)[1] > 1792:
            close = cam
            break
    assert close is not None, "no camera reaches the long-list sort path"
    empty = ref_python.make_camera(_camera(0, W, H, away=True), cuda_device)
    assert _strand_max_tile_len(hair, ordinary, W, H)[1] <= 1792
    Rs = {n: _eager_R(pc, hair, c, pair.bg, W, H) for n, c in (("ordinary", ordinary), ("close", close), ("empty", empty))}
    assert Rs["empty"] == 0 and Rs["close"] > 0 and Rs["ordinary"] > 0
    pair.step.capacity = _C.capacity_for(max(Rs.values()))     # no overflow: every frame replays from the first graph
    gts = _gts(cuda_device, W, H)
    order = [ordinary, ordinary, close, ordinary, empty, close, empty, ordinary]
    for it, cam in enumerate(order):
        pair.run(it, cam, gts[it % 3])
    assert pair.step.captures == 1 and pair.step.overflows == 0 and pair.step.replays == len(order) - 2
    # the capturable render itself: image and radii equal to render_hair_strands' for all three cameras
    binning = _C.binning_workspace(pair.step.capacity, cuda_device)
    status = torch.zeros(1, dtype=torch.int32, device=cuda_device)
    with torch.no_grad():
        for cam in (ordinary, close, empty):
            pkg = renderer.render_hair_strands(cam, pc, hair, PIPE, pair.bg)
            img_c, radii_c = renderer.render_hair_strands_capturable(_static_camera(cam, cuda_device), pc, hair, pair.bg,
                                                                     W, H, binning, pair.step.capacity, status)
            assert torch.equal(pkg["raw"], img_c) and torch.equal(pkg["radii"], radii_c)
    assert int(status) == 0


def test_overflow_skips_then_reruns(cuda_device, det, monkeypatch):
    from gaussianhaircut_b200 import graphs
    W, H = 512, 512
    pair = _Pair(cuda_device, 300, 99, 20000, W, H)
    cams, gts = _cams(cuda_device, W, H), _gts(cuda_device, W, H)
    R0 = _eager_R(pair.eager[0], pair.eager[1], cams[0], pair.bg, W, H)
    seen = {}
    orig_eager, orig_policy = pair.step._eager, graphs.capacity_for
    monkeypatch.setattr(graphs, "capacity_for", lambda r: R0 // 2)      # the first capture: below every view's R

    def eager_after_replay(camera, gts_, dirs_grad):
        if pair.step.replays > 0 and "state" not in seen:
            seen["state"], seen["status"] = _state(*pair.capt[1:]), int(pair.step._host[0])
            monkeypatch.setattr(graphs, "capacity_for", orig_policy)
            pair.step.capacity = orig_policy(pair.step.r_max)
        return orig_eager(camera, gts_, dirs_grad)

    monkeypatch.setattr(pair.step, "_eager", eager_after_replay)
    it = 0
    while pair.step.replays == 0:                           # warm-ups, then the first (overflowing) replay
        before = _state(*pair.capt[1:]) if it > 0 else None
        pair.run(it, cams[it % 8], gts[it % 3])
        it += 1
    assert pair.step.overflows == 1 and seen["status"] & 1 and pair.step.capacity > R0
    for k in before:
        assert torch.equal(before[k], seen["state"][k]), f"the overflowed replay changed {k}"
    for it in range(it, it + 6):
        pair.run(it, cams[it % 8], gts[it % 3])
    assert pair.step.captures == 2 + (pair.step.overflows - 1) and pair.step.replays >= 5


def test_overflow_touches_no_record_beyond_capacity(cuda_device):
    """The capturable strand render on a frame whose R exceeds the capacity: status bit, guard bytes intact, the
    background image, zero radii and zero gradients."""
    from gaussianhaircut_b200 import _C, renderer
    W, H = 512, 512
    pc, hair, _ = _models(cuda_device, 300, 99, 20000, False)
    cam = ref_python.make_camera(_camera(0, W, H), cuda_device)
    bg = torch.tensor(synth.BG_DEFAULT, device=cuda_device)
    R = _eager_R(pc, hair, cam, bg, W, H)
    cap = R // 2
    nbytes = _C.binning_workspace(cap, cuda_device).numel()
    raw = torch.full((nbytes + 65536,), 0xA5, dtype=torch.uint8, device=cuda_device)
    binning, guard = raw[:nbytes], raw[nbytes:]
    status = torch.zeros(1, dtype=torch.int32, device=cuda_device)
    nr = torch.zeros(1, dtype=torch.int32, device=cuda_device)
    for d in (False, True):
        torch.use_deterministic_algorithms(d)
        try:
            for n in NAMES:
                getattr(hair, n).grad = None
            img, radii = renderer.render_hair_strands_capturable(_static_camera(cam, cuda_device), pc, hair, bg, W, H,
                                                                 binning, cap, status, nr)
            img.backward(synth.upstream_gradient(W, H, 0).to(cuda_device))
            torch.cuda.synchronize()
        finally:
            torch.use_deterministic_algorithms(False)
        assert int(status) == 1 and int(nr) == R
        assert not bool(radii.any())
        assert torch.equal(img, bg.view(-1, 1, 1).expand_as(img))
        for n in NAMES:
            assert not bool(getattr(hair, n).grad.any()), f"{n} gradient not zero (deterministic={d})"
    assert bool((guard == 0xA5).all()), "a kernel wrote beyond the binning buffer"


def test_dirs_grad(cuda_device, det):
    W, H = 512, 512
    pair = _Pair(cuda_device, 300, 99, 20000, W, H)
    cams, gts = _cams(cuda_device, W, H), _gts(cuda_device, W, H)
    gen = torch.Generator().manual_seed(21)
    shape = tuple(pair.eager[1]._dirs.shape)
    for it in range(8):
        prior = (1e-3 * torch.randn(shape, generator=gen)).to(cuda_device)
        pair.run(it, cams[it % 8], gts[it % 3], dirs_grad=prior)
    assert pair.step.replays == 8 - 2 and int(pair.capt[2].step_state[0]) == 8
    # a NaN in the prior gradient skips the step on both paths (the replay and, after it, the eager iteration)
    bad = (1e-3 * torch.randn(shape, generator=gen)).to(cuda_device)
    bad[3, 7, 1] = float("nan")
    before = _state(*pair.capt[1:])
    a, b = pair.run(8, cams[0], gts[0], dirs_grad=bad)
    for k in before:
        assert torch.equal(before[k], b[k]), f"a NaN prior gradient changed {k}"
    assert int(pair.step._nan_flag) == 0 and int(pair.nan) == 0
    pair.run(9, cams[1], gts[1], dirs_grad=(1e-3 * torch.randn(shape, generator=gen)).to(cuda_device))
    pair.run(10, cams[2], gts[2])                          # without a prior gradient: a new key, warm-ups, a new capture
    pair.run(11, cams[3], gts[0])
    pair.run(12, cams[4], gts[1])
    assert int(pair.capt[2].step_state[0]) == 12 and pair.step.captures == 2 + pair.step.overflows


def _rig(dev, W, H, n=8, seed=0):
    """A CameraRig on the synthetic ring with small residuals (pose and field of view)."""
    from gaussianhaircut_b200.cameras import CameraRig
    gen = torch.Generator().manual_seed(seed)
    base, res = [], []
    for k in range(n):
        d = synth.make_camera(8 * k, W, H, focal_factor=1.0 + 0.1 * k)
        base.append(torch.cat([d["world_view_transform"].T.reshape(16),
                               torch.tensor([float(d["FoVx"]), float(d["FoVy"])])]))
        res.append(torch.cat([0.01 * torch.randn(3, generator=gen), 0.005 * torch.randn(3, generator=gen),
                              0.05 * (torch.rand(2, generator=gen) - 0.5)]))
    return CameraRig(torch.stack(base).to(dev), torch.stack(res).to(dev), [f"view_{k:02d}" for k in range(n)],
                     [(W, H)] * n)


def test_frozen_rig_views(cuda_device, det):
    W, H = 512, 512
    rigs = (_rig(cuda_device, W, H), _rig(cuda_device, W, H))
    pair = _Pair(cuda_device, 300, 99, 20000, W, H, rigs=rigs)
    gts = _gts(cuda_device, W, H)
    for it in range(10):
        i = (3 * it) % 8
        pair.run(it, rigs[0].view(i, requires_grad=False), gts[it % 3], cam_c=rigs[1].view(i))
    assert pair.step.replays == 10 - 2 and pair.step.captures == 1 + pair.step.overflows
    assert torch.equal(rigs[0].residuals.detach(), rigs[1].residuals.detach()) and not bool(rigs[1].touched.any())


def test_refusals(cuda_device):
    from gaussianhaircut_b200 import projection
    from gaussianhaircut_b200.graphs import CapturedStrandStep
    W, H = 256, 192
    pc, hair, opt = _models(cuda_device, 50, 20, 2000, True)
    bg = torch.tensor(synth.BG_DEFAULT, device=cuda_device)
    with pytest.raises(RuntimeError, match="debug"):
        CapturedStrandStep(pc, hair, opt, W, H, bg, LAMBDAS, pipe=types.SimpleNamespace(debug=True))
    with pytest.raises(RuntimeError, match="capturable=True"):
        CapturedStrandStep(pc, hair, _models(cuda_device, 50, 20, 2000, False)[2], W, H, bg, LAMBDAS)
    prev = projection.set_gradient_arena(torch.zeros(1024, device=cuda_device))
    try:
        with pytest.raises(RuntimeError, match="gradient arena"):
            CapturedStrandStep(pc, hair, opt, W, H, bg, LAMBDAS)
    finally:
        projection.set_gradient_arena(prev)
    step = CapturedStrandStep(pc, hair, opt, W, H, bg, LAMBDAS)
    gt = _gts(cuda_device, W, H, 1)[0]
    x0 = hair._dirs.detach().clone()
    cam = ref_python.make_camera(_camera(0, W, H), cuda_device, trainable=True)
    with pytest.raises(RuntimeError, match="trainable cameras"):
        step.step(cam, *gt)
    prev = projection.set_gradient_arena(torch.zeros(1024, device=cuda_device))
    try:
        with pytest.raises(RuntimeError, match="gradient arena"):
            step.step(ref_python.make_camera(_camera(0, W, H), cuda_device), *gt)
    finally:
        projection.set_gradient_arena(prev)
    with pytest.raises(RuntimeError, match="shape of _dirs"):
        step.step(ref_python.make_camera(_camera(0, W, H), cuda_device), *gt, dirs_grad=torch.zeros(3, device=cuda_device))
    assert step.captures == 0 and step._warm == 0 and torch.equal(hair._dirs.detach(), x0)
    assert int(opt.step_state[0]) == 0
