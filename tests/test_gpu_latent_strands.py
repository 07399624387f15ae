"""GPU tests of the latent strand stage on the fused path (renderer.render_hair_segments, its capturable form, the
gh_hair_segments_*_capturable entry points and graphs.CapturedLatentStrandStep):

  * render_hair_segments against the reference's own initialize_gaussians_hair()-built GaussianModelHair and
    render_hair() on the reference's rasterizer build: maps, radii, viewspace gradients and the gradients of the five
    segment tensors (and, with `_xyz` and `_dir` formed from a polyline leaf `p` by the reference's expressions, of
    `p`); and against this package's render_hair on the same inputs;
  * captured equals eager: 12 iterations over 8 cameras with different fields of view, a stand-in decoder with
    torch.optim.AdamW outside the graph, in deterministic mode: after every iteration every network parameter, the
    AdamW state and the 8 losses are equal bit for bit, for both loss-option pairs and hair only;
  * one graph serves a camera on the long-list sort path, an ordinary one and one that sees nothing; overflow leaves
    the guard bytes past the binning buffer intact, reruns eagerly, recaptures and stays bit-identical; frozen
    CameraRig views; a backward that reaches the gradients of an earlier step raises.
"""
import os
import sys
import types

import pytest
import torch

import _util
from _latent_strands import StandInDecoder, polyline as _polyline
from _util import rel_err

sys.path.insert(0, os.path.join(_util.ROOT, "oracle"))
import ref_python  # noqa: E402
import synth  # noqa: E402

pytestmark = pytest.mark.gpu
REL_TOL = 1e-4
LAMBDAS = (0.1, 1.0, 0.1)             # lambda_dl1, lambda_dmask, lambda_dorient
LAMBDA_DSDS = 0.05
PIPE = types.SimpleNamespace(debug=False)
OPTIONS = [(True, True), (False, False)]


@pytest.fixture
def det():
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(prev, warn_only=warn)


def _need_reference():
    if not ref_python.available() or not _util.ref_available():
        pytest.skip("reference Python sources / oracle/_ref not staged")


def _weights(H, W, device, seed):
    g = torch.Generator().manual_seed(seed)
    return {k: torch.rand(c, H, W, generator=g).to(device) for k, c in (("render", 3), ("mask", 2), ("orient_angle", 1),
                                                                          ("orient_conf", 1))}


def _loss(pkg, Wt):
    return sum((pkg[k] * Wt[k]).sum() for k in Wt)


def _head(n_head):
    if n_head:
        return synth.make_blob_scene(n_head, seed=2, spread=0.08, max_scale=0.004)
    s = synth.make_blob_scene(1, seed=0)
    return {k: v[:0] for k, v in s.items()}


def _from_polyline(hair, p):
    """generate_strands' expressions (gaussian_model_latent_strands.py:453-454) and initialize_gaussians_hair's
    rotation (:489-498) on a leaf polyline `p`."""
    from utils.general_utils import parallel_transport
    hair._xyz = (p[:, 1:] + p[:, :-1]).view(-1, 3) * 0.5
    hair._dir = (p[:, 1:] - p[:, :-1]).view(-1, 3)
    ex = torch.cat([torch.ones_like(hair._xyz[:, :1]), torch.zeros_like(hair._xyz[:, :2])], dim=-1)
    hair._rotation = parallel_transport(a=ex, b=hair._dir).view(-1, 4)


@pytest.mark.parametrize("S, n_head, W, H, polyline", [(2000, 20000, 512, 384, False), (10000, 200000, 1920, 1080, False),
                                                      (2000, 20000, 512, 384, True)],
                         ids=["2000x99+head-512x384", "10000x99+head-1080p", "polyline-leaf-512x384"])
def test_render_hair_segments_matches_the_reference_pipeline(cuda_device, S, n_head, W, H, polyline):
    """render_hair_segments against the reference's GaussianModelHair (rotations from initialize_gaussians_hair) and
    render_hair on the reference's rasterizer; the same inputs through this package's render_hair for the record."""
    _need_reference()
    from gaussianhaircut_b200 import renderer
    head = _head(n_head)
    hair_scene = synth.make_strand_scene(S, seed=4, segments=99)
    cam_d = synth.make_camera(7, W, H)
    bg = torch.tensor(synth.BG_DEFAULT, device=cuda_device)
    Wt = _weights(H, W, cuda_device, 9)
    ref_mod = ref_python.load_renderer("ref")
    res = {}
    for which, fn in (("segments", renderer.render_hair_segments), ("ref", ref_mod.render_hair),
                      ("render_hair", renderer.render_hair)):
        pc, pc_hair = ref_python.make_hair_models(head, hair_scene, cuda_device)
        p = None
        if polyline:
            p = _polyline(hair_scene, S).to(cuda_device).requires_grad_(True)
            _from_polyline(pc_hair, p)
        cam = ref_python.make_camera(cam_d, cuda_device, trainable=True)
        pkg = fn(cam, pc, pc_hair, ref_python.pipe(), bg)
        if polyline:
            for name in ref_python.HAIR_PARAMS:
                getattr(pc_hair, name).retain_grad()
        _loss(pkg, Wt).backward()
        torch.cuda.synchronize()
        res[which] = (pkg, pc_hair, cam, p)
    (pa, ha, ca, p_a), (pb, hb, cb, p_b) = res["segments"], res["ref"]
    P = pb["visibility_filter"].numel()
    assert pa["visibility_filter"].numel() == P
    assert int((pa["visibility_filter"] != pb["visibility_filter"]).sum()) <= max(2, P // 100000)
    assert int((pa["radii"] != pb["radii"]).sum()) <= max(4, P // 20000)          # ceil ties
    for k in ("render", "mask", "orient_conf"):
        assert rel_err(pa[k], pb[k]) <= REL_TOL, f"{k}: {rel_err(pa[k], pb[k])}"
    assert rel_err(pa["orient_angle"], pb["orient_angle"]) <= 1e-3
    for name in ref_python.HAIR_PARAMS:
        ga, gb = getattr(ha, name).grad, getattr(hb, name).grad
        assert ga is not None and gb is not None, name
        assert ga.shape == gb.shape, name
        assert rel_err(ga, gb) <= 2 * REL_TOL, f"{name}: {rel_err(ga, gb)}"
    if polyline:
        assert rel_err(p_a.grad, p_b.grad) <= 2 * REL_TOL, f"p: {rel_err(p_a.grad, p_b.grad)}"
    for name in ("world_view_transform", "full_proj_transform", "camera_center"):
        assert rel_err(getattr(ca, name).grad, getattr(cb, name).grad) <= 2 * REL_TOL, name
    assert rel_err(pa["viewspace_points"].grad, pb["viewspace_points"].grad) <= 2 * REL_TOL
    # against today's path (render_hair: PyTorch-built rotations and get_scaling): report the measured difference
    pr, hr = res["render_hair"][0], res["render_hair"][1]
    diffs = {k: rel_err(pa[k], pr[k]) for k in ("render", "mask", "orient_conf")}
    diffs.update({name: rel_err(getattr(ha, name).grad, getattr(hr, name).grad) for name in ref_python.HAIR_PARAMS})
    if polyline:
        diffs["p"] = rel_err(p_a.grad, res["render_hair"][3].grad)
    print(f"render_hair_segments vs render_hair, norm-relative ({S}x99 + {n_head} head, {W}x{H}):", diffs)
    for k, e in diffs.items():
        assert e <= 2 * REL_TOL, f"{k}: {e}"


# ------------------------------------------------------------------------------------------------ captured vs eager
def _models(dev, S, L, n_head):
    from gaussianhaircut_b200 import renderer
    pc = ref_python.make_hair_models(_head(n_head), synth.make_strand_scene(1, seed=0, segments=1), dev)[0] if n_head \
        else None
    if pc is not None:
        renderer._head_block(pc)
    dec = StandInDecoder(S, L, seed=4).to(dev)
    hair = types.SimpleNamespace(scale=2e-4 * torch.ones(1, device=dev), active_sh_degree=3)
    opt = torch.optim.AdamW(dec.parameters(), lr=1e-3)
    return pc, dec, hair, opt


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


def _ldf(diffusion_dict, like):
    """train_latent_strands.py:140-145 for the prior term."""
    LDF = diffusion_dict.get("L_diff")
    LDF = LDF if LDF is not None else torch.zeros_like(like)
    return torch.zeros_like(like) if bool(torch.isnan(LDF).any()) else LDF


def _eager_step(pc, dec, hair, opt, cam, gt, bg, options):
    """The train_latent_strands.py iteration on this package's eager path."""
    from gaussianhaircut_b200 import losses as ghl, renderer
    dd = dec.generate(hair)
    pkg = renderer.render_hair_segments(cam, pc, hair, PIPE, bg)
    total, l8 = ghl.HairImageLoss.apply(pkg["raw"], *gt, LAMBDAS[0], 0.0, LAMBDAS[1], LAMBDAS[2], "latent_strands", *options)
    (total + _ldf(dd, total) * LAMBDA_DSDS).backward()
    opt.step()
    opt.zero_grad(set_to_none=True)
    return l8.detach().cpu()


def _captured_step(step, dec, hair, opt, cam, gt):
    dd = dec.generate(hair)
    loss, l8 = step.step(cam, *gt, hair)
    (loss + _ldf(dd, loss) * LAMBDA_DSDS).backward()
    opt.step()
    opt.zero_grad(set_to_none=True)
    return l8


def _state(dec, opt):
    out = {}
    for n, p in dec.named_parameters():
        out[n] = p.detach().clone()
        for k, v in opt.state[p].items():
            out[f"{n}.{k}"] = v.clone() if isinstance(v, torch.Tensor) else torch.tensor(v)
    return out


class _Pair:
    """An eager decoder and a captured one from the same initialisation, stepped on the same inputs."""

    def __init__(self, dev, S, L, n_head, W, H, options=(True, True), capacity=None, rigs=None):
        from gaussianhaircut_b200.graphs import CapturedLatentStrandStep
        self.options = options
        self.eager = _models(dev, S, L, n_head)
        self.capt = _models(dev, S, L, n_head)
        self.bg = torch.tensor(synth.BG_DEFAULT, device=dev)
        self.step = CapturedLatentStrandStep(self.capt[0], W, H, self.bg, LAMBDAS, use_gt_orient_conf=options[0],
                                             train_orient_conf=options[1], capacity=capacity,
                                             cameras=None if rigs is None else rigs[1])

    def run(self, it, cam, gt, cam_c=None):
        le = _eager_step(*self.eager, cam, gt, self.bg, self.options)
        pc, dec, hair, opt = self.capt
        lc = _captured_step(self.step, dec, hair, opt, cam if cam_c is None else cam_c, gt)
        torch.cuda.synchronize()
        a, b = _state(*self.eager[1:4:2]), _state(*self.capt[1:4:2])
        assert torch.equal(le, lc), f"iteration {it}: losses {le} vs {lc}"
        assert a.keys() == b.keys()
        for k in a:
            assert a[k].shape == b[k].shape and torch.equal(a[k], b[k]), f"iteration {it}: {k}"
        return a, b


@pytest.mark.parametrize("S, L, n_head, W, H, options", [(300, 99, 20000, 512, 512, (True, True)),
                                                         (300, 99, 20000, 512, 512, (False, False)),
                                                         (1000, 32, 0, 250, 187, (True, True))],
                         ids=["head_512_gt_conf", "head_512_unit_weights_no_conf", "hair_only_250x187"])
def test_captured_equals_eager(cuda_device, det, S, L, n_head, W, H, options):
    pair = _Pair(cuda_device, S, L, n_head, W, H, options)
    cams, gts = _cams(cuda_device, W, H), _gts(cuda_device, W, H)
    for it in range(12):
        pair.run(it, cams[it % 8], gts[it % 3])
    assert pair.step.replays == 12 - 2 and pair.step.captures == 1 + pair.step.overflows


def _segment_max_tile_len(hair, cam, W, H):
    """(R, longest tile list) of the segment rows alone."""
    from gaussianhaircut_b200 import projection, renderer
    pi = projection.pack_inputs(hair._xyz, hair.scale, None, hair._dir, hair._features_dc, hair._features_rest, None, None,
                                hair._orient_conf, cam.world_view_transform, cam.full_proj_transform, cam.camera_center,
                                renderer._tan_half(cam.FoVx), renderer._tan_half(cam.FoVy), W, H, 3, 1.0,
                                projection.HAIR_STRANDS)
    _o, _r, _g, _i, R, max_len = projection.project_forward_binned(pi)
    return R, max_len


def _eager_R(pc, hair, cam, bg, W, H):
    from gaussianhaircut_b200 import _C, renderer
    with torch.no_grad():
        pkg = renderer.render_hair_segments(cam, pc, hair, PIPE, bg)
    return _C.last_num_rendered((bg.device.index, int(pkg["radii"].shape[0]), W, H))


def _static_camera(cam, dev):
    from gaussianhaircut_b200 import renderer
    return {"viewmatrix": cam.world_view_transform, "projmatrix": cam.full_proj_transform, "campos": cam.camera_center,
            "tan_fov": torch.tensor([renderer._tan_half(cam.FoVx), renderer._tan_half(cam.FoVy)], device=dev)}


def test_one_graph_long_lists_and_empty_frame(cuda_device, det):
    from gaussianhaircut_b200 import _C, renderer
    W, H = 512, 512
    pair = _Pair(cuda_device, 300, 99, 20000, W, H)
    pc, dec, hair, _ = pair.eager
    with torch.no_grad():
        dec.generate(hair)
    ordinary = ref_python.make_camera(_camera(0, W, H), cuda_device)
    close = None                  # far enough away that the model falls into a few tiles: lists beyond 1792 records
    for radius in (3.0, 6.0, 12.0, 24.0):
        cam = ref_python.make_camera(_camera(0, W, H, radius=radius), cuda_device)
        if _segment_max_tile_len(hair, cam, W, H)[1] > 1792:
            close = cam
            break
    assert close is not None, "no camera reaches the long-list sort path"
    empty = ref_python.make_camera(_camera(0, W, H, away=True), cuda_device)
    assert _segment_max_tile_len(hair, ordinary, W, H)[1] <= 1792
    Rs = {n: _eager_R(pc, hair, c, pair.bg, W, H) for n, c in (("ordinary", ordinary), ("close", close), ("empty", empty))}
    assert Rs["empty"] == 0 and Rs["close"] > 0 and Rs["ordinary"] > 0
    # no overflow: every frame replays from the first graph (twice the largest R: the decoder moves the strands)
    pair.step.capacity = _C.capacity_for(2 * max(Rs.values()))
    gts = _gts(cuda_device, W, H)
    order = [ordinary, ordinary, close, ordinary, empty, close, empty, ordinary]
    for it, cam in enumerate(order):
        pair.run(it, cam, gts[it % 3])
    assert pair.step.captures == 1 and pair.step.overflows == 0 and pair.step.replays == len(order) - 2
    # the capturable render itself: image and radii equal to render_hair_segments' for all three cameras
    binning = _C.binning_workspace(pair.step.capacity, cuda_device)
    status = torch.zeros(1, dtype=torch.int32, device=cuda_device)
    with torch.no_grad():
        dec.generate(hair)
        for cam in (ordinary, close, empty):
            pkg = renderer.render_hair_segments(cam, pc, hair, PIPE, pair.bg)
            img_c, radii_c = renderer.render_hair_segments_capturable(_static_camera(cam, cuda_device), pc, hair, pair.bg,
                                                                      W, H, binning, pair.step.capacity, status)
            assert torch.equal(pkg["raw"], img_c) and torch.equal(pkg["radii"], radii_c)
    assert int(status) == 0


def test_overflow_skips_then_reruns(cuda_device, det, monkeypatch):
    from gaussianhaircut_b200 import graphs
    W, H = 512, 512
    pair = _Pair(cuda_device, 300, 99, 20000, W, H)
    cams, gts = _cams(cuda_device, W, H), _gts(cuda_device, W, H)
    pc, dec, hair, _ = pair.eager
    with torch.no_grad():
        dec.generate(hair)
    R0 = _eager_R(pc, hair, cams[0], pair.bg, W, H)
    seen = {}
    orig_eager, orig_policy = pair.step._eager, graphs.capacity_for
    monkeypatch.setattr(graphs, "capacity_for", lambda r: R0 // 2)      # the first capture: below every view's R

    def eager_after_replay(camera, gts_, pc_hair):
        if pair.step.replays > 0 and "status" not in seen:
            seen["status"] = int(pair.step._host[0])
            monkeypatch.setattr(graphs, "capacity_for", orig_policy)
            pair.step.capacity = orig_policy(pair.step.r_max)
        return orig_eager(camera, gts_, pc_hair)

    monkeypatch.setattr(pair.step, "_eager", eager_after_replay)
    it = 0
    while pair.step.replays == 0:                           # warm-ups, then the first (overflowing) replay
        pair.run(it, cams[it % 8], gts[it % 3])
        it += 1
    assert pair.step.overflows == 1 and seen["status"] & 1 and pair.step.capacity > R0
    for it in range(it, it + 6):
        pair.run(it, cams[it % 8], gts[it % 3])
    assert pair.step.captures == 2 + (pair.step.overflows - 1) and pair.step.replays >= 5


def test_overflow_touches_no_record_beyond_capacity(cuda_device):
    """The capturable segment render on a frame whose R exceeds the capacity: status bit, guard bytes intact, the
    background image, zero radii and zero gradients."""
    from gaussianhaircut_b200 import _C, renderer
    W, H = 512, 512
    pc, dec, hair, _ = _models(cuda_device, 300, 99, 20000)
    cam = ref_python.make_camera(_camera(0, W, H), cuda_device)
    bg = torch.tensor(synth.BG_DEFAULT, device=cuda_device)
    with torch.no_grad():
        dec.generate(hair)
    R = _eager_R(pc, hair, cam, bg, W, H)
    cap = R // 2
    nbytes = _C.binning_workspace(cap, cuda_device).numel()
    raw = torch.full((nbytes + 65536,), 0xA5, dtype=torch.uint8, device=cuda_device)
    binning, guard = raw[:nbytes], raw[nbytes:]
    status = torch.zeros(1, dtype=torch.int32, device=cuda_device)
    nr = torch.zeros(1, dtype=torch.int32, device=cuda_device)
    names = ("_xyz", "_dir", "_features_dc", "_features_rest", "_orient_conf")
    for d in (False, True):
        torch.use_deterministic_algorithms(d)
        try:
            leaves = types.SimpleNamespace(scale=hair.scale, active_sh_degree=3,
                                           **{n: getattr(hair, n).detach().clone().requires_grad_(True) for n in names})
            img, radii = renderer.render_hair_segments_capturable(_static_camera(cam, cuda_device), pc, leaves, bg, W, H,
                                                                  binning, cap, status, nr)
            img.backward(synth.upstream_gradient(W, H, 0).to(cuda_device))
            torch.cuda.synchronize()
        finally:
            torch.use_deterministic_algorithms(False)
        assert int(status) == 1 and int(nr) == R
        assert not bool(radii.any())
        assert torch.equal(img, bg.view(-1, 1, 1).expand_as(img))
        for n in names:
            assert not bool(getattr(leaves, n).grad.any()), f"{n} gradient not zero (deterministic={d})"
    assert bool((guard == 0xA5).all()), "a kernel wrote beyond the binning buffer"


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


def test_stale_backward_raises(cuda_device):
    from gaussianhaircut_b200.graphs import CapturedLatentStrandStep
    W, H = 256, 192
    pc, dec, hair, opt = _models(cuda_device, 100, 20, 2000)
    bg = torch.tensor(synth.BG_DEFAULT, device=cuda_device)
    step = CapturedLatentStrandStep(pc, W, H, bg, LAMBDAS)
    cams, gts = _cams(cuda_device, W, H), _gts(cuda_device, W, H, 1)
    for it in range(4):                                  # warm-ups, capture, replay: both paths
        dec.generate(hair)
        loss_a, _ = step.step(cams[it], *gts[0], hair)
        dec.generate(hair)
        loss_b, _ = step.step(cams[it + 1], *gts[0], hair)
        with pytest.raises(RuntimeError, match="overwritten"):
            loss_a.backward()
        loss_b.backward()
        assert dec.p.grad is not None and bool(dec.p.grad.abs().sum() > 0)
        opt.zero_grad(set_to_none=True)
    assert step.captures >= 1 and step.replays >= 1
