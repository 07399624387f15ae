"""GPU tests of the deterministic blend backward, selected by torch.use_deterministic_algorithms(True):

  * reproducible: on the 1080p strand bench scene, repeated runs -- one of them with a side stream keeping the GPU busy --
    give bit-identical gradients and accumulation records on the 9-tensor, arena and records + projection paths, and
    through render_hair_strands with a head block;
  * correct: the float64 replay scenes of test_gpu_blend_replay.py pass at the same TOL with the switch on, and the
    deterministic gradients agree with the default path's;
  * edges: nothing rendered, a Gaussian over every tile, lists on the long-list sort path, odd image sizes, early stops;
  * end to end: a short training loop with densification, run twice from the same seed, ends bit-identical;
  * the image loss, whose sums go through no atomics under the switch, is bit-identical across calls.
"""
import os
import sys
import types

import numpy as np
import pytest
import torch

import _util
import test_gpu_blend_replay as rep

sys.path.insert(0, os.path.join(_util.ROOT, "oracle"))
import ref_python  # noqa: E402
import synth  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture
def det():
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(prev, warn_only=warn)


def _mine():
    import gaussianhaircut_b200._C as mine
    return mine


def acc16(geom: torch.Tensor, P: int) -> torch.Tensor:
    """The (P, 16) accumulation records inside a geometry workspace (GhGeomWS::carve: 256-byte aligned segments)."""
    a = lambda n: (n + 255) // 256 * 256  # noqa: E731
    off = a(P * 32) + a(P * 4)
    return geom[off:off + 64 * P].view(torch.float32).view(P, 16).clone()


# ------------------------------------------------------------------------------------------------- bench scene
_SCENE = {}


def bench_views(device):
    if "v" not in _SCENE:
        scene = synth.make_strand_scene(5000, seed=0)              # 500 000 Gaussians, the bench.py default
        _SCENE["v"] = [synth.rasterizer_inputs(scene, synth.make_camera(k, 1920, 1080), mode=m, device=device)
                       for k, m in ((0, "native"), (8, "render"))]
        _SCENE["dL"] = synth.upstream_gradient(1920, 1080, 0).to(device)
    return _SCENE["v"], _SCENE["dL"]


def _busy_side_stream(device):
    """Queue ~20 ms of unrelated kernels on another stream: the backward's CTAs share the SMs with them."""
    s = torch.cuda.Stream(device)
    x = torch.rand(1 << 24, device=device)
    with torch.cuda.stream(s):
        for _ in range(60):
            x.mul_(1.0000001).add_(1e-7)
    return s, x


def _run_native(inp, dL, path, busy):
    mod = _mine()
    r = mod.rasterize_gaussians(*_util.native_args(inp))
    bw = _util.backward_args(inp, r[2], dL, r[3], r[0], r[4], r[5])
    side = _busy_side_stream(dL.device) if busy else None
    if path == "tensors":
        out = list(mod.rasterize_gaussians_backward(*bw))
    elif path == "arena":
        flat, _g, _sh = mod.rasterize_gaussians_backward_arena(*bw)
        out = [flat]
    else:                                   # records mode + the projection backward reading them in place
        kw, s = inp["kwargs"], inp["settings"]
        mod.rasterize_gaussians_backward_records(s["bg"], kw["means3D"], r[2], kw["colors_precomp"], kw["conic_precomp"],
                                                 s["viewmatrix"], s["projmatrix"], s["tanfovx"], s["tanfovy"], dL,
                                                 s["campos"], r[3], r[0], r[4], r[5], False)
        out = []
    torch.cuda.synchronize()
    if side is not None:
        side[0].synchronize()
    P = inp["kwargs"]["means3D"].shape[0]
    return [t.clone() for t in out] + [acc16(r[3], P)]


@pytest.mark.parametrize("path", ["tensors", "arena", "records"])
def test_bench_scene_is_bit_reproducible(cuda_device, det, path):
    views, dL = bench_views(cuda_device)
    inp = views[1] if path == "records" else views[0]              # the records mode needs the conic call shape
    runs = [_run_native(inp, dL, path, busy=(k == 2)) for k in range(5)]
    for k, r in enumerate(runs[1:], 1):
        for a, b in zip(runs[0], r):
            assert torch.equal(a, b), f"run {k} differs from run 0 ({path})"
    assert float(runs[0][-1].abs().sum()) > 0


def test_bench_scene_default_and_det_agree(cuda_device):
    views, dL = bench_views(cuda_device)
    fast = _run_native(views[0], dL, "tensors", busy=False)
    torch.use_deterministic_algorithms(True)
    try:
        slow = _run_native(views[0], dL, "tensors", busy=False)
    finally:
        torch.use_deterministic_algorithms(False)
    for n, a, b in zip(_util.GRAD_NAMES, fast, slow):
        assert _util.rel_err(b, a) <= 1e-5, f"{n}: {_util.rel_err(b, a)}"


def _strand_models(dev, S=300, L=33, n_head=20000):
    import _strands
    poly = _strands.make_strand_polylines(S, L, seed=4)
    hair = types.SimpleNamespace(active_sh_degree=3, max_sh_degree=3, pts_origins=poly["origins"].to(dev),
                                 scale=poly["scale"] * torch.ones(1, device=dev))
    for n, k in (("_dirs", "dirs"), ("_features_dc", "f_dc"), ("_features_rest", "f_rest"), ("_orient_conf", "conf")):
        setattr(hair, n, torch.nn.Parameter(poly[k].to(dev).contiguous()))
    h = synth.make_blob_scene(n_head, seed=2, spread=0.08, max_scale=0.004)
    g = torch.Generator().manual_seed(3)
    head = types.SimpleNamespace(
        xyz_precomp=h["xyz"].to(dev), scaling_precomp=h["scaling"].to(dev),
        rotation_precomp=torch.nn.functional.normalize(h["rotation"], dim=1).to(dev),
        opacity_precomp=h["opacity"].reshape(-1, 1).to(dev),
        shs_view=(0.3 * torch.randn(n_head, 3, 16, generator=g)).to(dev))
    return head, hair


def test_render_hair_strands_with_head_block_is_bit_reproducible(cuda_device, det):
    from gaussianhaircut_b200 import renderer
    cam = ref_python.make_camera(synth.make_camera(7, 512, 512), cuda_device)
    bg = torch.tensor(synth.BG_DEFAULT, device=cuda_device)
    Wt = torch.rand(10, 512, 512, generator=torch.Generator().manual_seed(9)).to(cuda_device)
    head, hair = _strand_models(cuda_device)
    res = []
    for k in range(3):
        for p in (hair._dirs, hair._features_dc, hair._features_rest, hair._orient_conf):
            p.grad = None
        side = _busy_side_stream(cuda_device) if k == 1 else None
        pkg = renderer.render_hair_strands(cam, head, hair, types.SimpleNamespace(debug=False), bg)
        torch.cat([pkg["render"], pkg["mask"], pkg["orient_conf"]]).mul(Wt[:6]).sum().backward()
        torch.cuda.synchronize()
        if side is not None:
            side[0].synchronize()
        res.append([hair._dirs.grad.clone(), hair._features_dc.grad.clone(), hair._orient_conf.grad.clone(),
                    pkg["viewspace_points"].grad.clone()])
    assert float(res[0][0].abs().sum()) > 0
    for r in res[1:]:
        for a, b in zip(res[0], r):
            assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------- correctness + edges
REPLAY_SCENES = {
    "border-33x17": lambda: rep.border_scene(33, 17), "border-47x31": lambda: rep.border_scene(47, 31),
    "alpha-band": rep.band_scene, "early-stop": rep.stop_scene,
    **{f"window-{n}" + (f"-stop{s}" if s else ""): (lambda n=n, s=s: rep.window_scene(n, s)) for n, s in rep.WINDOW_CASES},
    **{f"sort-{a}-{b}": (lambda a=a, b=b: rep.two_tile_scene(a, b)) for a, b in rep.SORT_CASES},
    "equal-depths-1000": lambda: rep.equal_depth_scene(1000), "equal-depths-3000": lambda: rep.equal_depth_scene(3000),
}


def _twice(inp, device):
    """check() with the switch on, twice: bit-identical, within TOL of the replay."""
    torch.use_deterministic_algorithms(True)
    try:
        w1, rp, o1 = rep.check(_mine(), inp, device)
        _w2, _rp, o2 = rep.check(_mine(), inp, device)
    finally:
        torch.use_deterministic_algorithms(False)
    for n in _util.GRAD_NAMES:
        assert torch.equal(o1["grads"][n], o2["grads"][n]), n
    rep.assert_within(w1)
    return rp, o1


@pytest.mark.parametrize("name", list(REPLAY_SCENES))
def test_replay_scenes_with_the_switch_on(cuda_device, name):
    inp = REPLAY_SCENES[name]()
    rp, o = _twice(inp, cuda_device)
    _wf, _rpf, of = rep.check(_mine(), inp, cuda_device)          # the default path on the same scene
    for n in _util.GRAD_NAMES:
        assert _util.rel_err(o["grads"][n], of["grads"][n]) <= 1e-5, n


def test_tile_ends_before_its_list(cuda_device):
    """Four wide, nearly opaque Gaussians in front of 40 faint ones: every pixel stops on the fourth, so the tile's
    walk ends at list position 3 and the rows of the 41 instances behind are the zero tail the CTA writes.  Unwritten
    rows would show up: under the switch torch fills fresh allocations with NaN."""
    n = 44
    rng = np.random.default_rng(12)
    px, py = 8.0 + rng.uniform(-0.5, 0.5, n), 8.0 + rng.uniform(-0.5, 0.5, n)
    con = rep.conics(np.full(n, 200.0), np.full(n, 150.0), rng.uniform(0, np.pi, n))
    op = np.concatenate([np.full(4, 0.95), np.full(n - 4, 0.3)])
    inp = rep.screen_scene(16, 16, px, py, 0.5 + 1e-4 * np.arange(n), con, op, seed=13)
    rp, o = _twice(inp, cuda_device)
    assert int(rp["n_contrib"].max()) == 3 and bool(rp["stopped"].all())
    for name in _util.GRAD_NAMES:
        g = o["grads"][name]
        if g.shape[0] == n and g.numel():
            assert not bool(g[3:].any()), name


def test_gaussian_over_every_tile(cuda_device):
    W, H = 160, 96
    rng = np.random.default_rng(5)
    n = 200
    px, py = rng.uniform(0, W, n), rng.uniform(0, H, n)
    con = rep.conics(rng.uniform(1, 6, n), rng.uniform(0.7, 3, n), rng.uniform(0, np.pi, n))
    px[0], py[0], con[0] = W / 2, H / 2, rep.conics(np.array([70.0]), np.array([45.0]), np.array([0.3]))[0]
    op = rng.uniform(0.1, 0.9, n)
    op[0] = 0.5
    inp = rep.screen_scene(W, H, px, py, rep.distinct_depths(n, rng), con, op, seed=8)
    rp, o = _twice(inp, cuda_device)
    rg = o["state"]["ranges"].view(np.uint32).reshape(-1, 2)
    T = ((W + 15) // 16) * ((H + 15) // 16)
    plist = o["state"]["point_list"].view(np.uint32)
    assert all(0 in plist[a:b] for a, b in rg[:T]), "Gaussian 0 must be listed in every tile"


def _nothing_rendered(P):
    """P Gaussians in front of the image but closer than the near plane (view depth 0.1 <= 0.2): all culled, R = 0."""
    rng = np.random.default_rng(4)
    px, py = rng.uniform(0, 64, P), rng.uniform(0, 48, P)
    return rep.screen_scene(64, 48, px, py, np.full(P, 0.1), np.tile(rep.TINY, (P, 1)), np.full(P, 0.5), seed=10)


@pytest.mark.parametrize("P", [0, 50])
def test_nothing_rendered(cuda_device, det, P):
    inp = rep.on(_nothing_rendered(P), cuda_device)
    mod = _mine()
    r = mod.rasterize_gaussians(*_util.native_args(inp))
    assert r[0] == 0
    dL = synth.upstream_gradient(64, 48, 0).to(cuda_device)
    g = mod.rasterize_gaussians_backward(*_util.backward_args(inp, r[2], dL, r[3], r[0], r[4], r[5]))
    torch.cuda.synchronize()
    for t in g:
        assert t.shape[0] == P and not bool(t.any())


def test_all_culled_but_one_tile_rendered(cuda_device):
    """Most Gaussians culled (radius 0, zero-area rectangle): their records come out zero from the gather."""
    W, H = 48, 32
    rng = np.random.default_rng(2)
    n = 64
    px, py = rng.uniform(-3000, -2000, n), rng.uniform(-3000, -2000, n)          # far off screen: not rendered
    px[:3], py[:3] = 8.0, 8.0
    con = np.tile(rep.TINY, (n, 1))
    inp = rep.screen_scene(W, H, px, py, rep.distinct_depths(n, rng), con, np.full(n, 0.5), seed=9)
    rp, o = _twice(inp, cuda_device)
    assert (o["radii"] > 0).sum() == 3
    for name in ("dL_dcolors", "dL_dopacity", "dL_dmeans2D"):
        assert not bool(o["grads"][name][3:].any())


# ------------------------------------------------------------------------------------------------- end to end
def _train(device, iters=30, strands=500, W=960, H=540):
    from gaussianhaircut_b200 import renderer, losses as ghl, densify
    from gaussianhaircut_b200.optim import FusedAdam
    scene = synth.make_strand_scene(strands, seed=0)                # 50 000 Gaussians
    raw = synth.raw_params_from_scene(scene, "gaussian_model")
    names = ("_xyz", "_features_dc", "_features_rest", "_opacity", "_label", "_scaling", "_rotation", "_orient_conf")
    keys = ("xyz", "f_dc", "f_rest", "opacity", "label", "scaling", "rotation", "conf")
    gnames = ("xyz", "f_dc", "f_rest", "opacity", "label", "scaling", "rotation", "orient_conf")
    lrs = (1.6e-4, 2.5e-3, 2.5e-4, 5e-2, 2.5e-3, 5e-3, 1e-3, 1e-3)
    pc = types.SimpleNamespace(active_sh_degree=3, max_sh_degree=3, percent_dense=0.01)
    for n, k in zip(names, keys):
        setattr(pc, n, torch.nn.Parameter(raw[k].to(device).contiguous()))
    pc.optimizer = FusedAdam([{"params": [getattr(pc, n)], "lr": lr, "name": g} for n, g, lr in zip(names, gnames, lrs)],
                             eps=1e-15)
    P0 = pc._xyz.shape[0]
    pc.xyz_gradient_accum = torch.zeros(P0, 1, device=device)
    pc.denom = torch.zeros(P0, 1, device=device)
    pc.max_radii2D = torch.zeros(P0, device=device)
    cams = [ref_python.make_camera(synth.make_camera(k, W, H), device) for k in range(0, 64, 8)]
    gen = torch.Generator().manual_seed(11)
    gt = (torch.rand(3, H, W, generator=gen).to(device), (torch.rand(2, H, W, generator=gen) > 0.3).float().to(device),
          torch.rand(1, H, W, generator=gen).to(device), torch.rand(1, H, W, generator=gen).to(device))
    bg = torch.tensor(synth.BG_DEFAULT, device=device)
    ws = torch.empty(ghl.workspace_elems(W, H), dtype=torch.float64, device=device)
    pipe = types.SimpleNamespace(debug=False)
    losses = []
    for it in range(iters):
        renders, radii, viewspace = renderer.render_raw(cams[it % len(cams)], pc, pipe, bg)
        l8, dL = ghl.image_loss_forward_backward(renders.detach(), *gt, 0.8, 0.2, 0.1, 0.1, workspace=ws)
        renders.backward(dL)
        with torch.no_grad():
            densify.update_max_radii(pc, radii)
            densify.add_densification_stats(pc, viewspace, radii > 0)
        pc.optimizer.step()
        pc.optimizer.zero_grad(set_to_none=True)
        if (it + 1) % 10 == 0:
            torch.manual_seed(1000 + it)
            torch.cuda.manual_seed(1000 + it)
            densify.densify_and_prune(pc, 2e-4, 0.005, 0.1, 20 if it > 15 else None)
        losses.append(l8.clone())
    torch.cuda.synchronize()
    out = {"loss": torch.stack(losses), "accum": pc.xyz_gradient_accum.clone(), "denom": pc.denom.clone(),
           "max_radii": pc.max_radii2D.clone()}
    for n in names:
        p = getattr(pc, n)
        out[n] = p.detach().clone()
        st = pc.optimizer.state[p]
        out[n + ".exp_avg"], out[n + ".exp_avg_sq"] = st["exp_avg"].clone(), st["exp_avg_sq"].clone()
    return out


def test_training_loop_is_bit_reproducible(cuda_device, det):
    a = _train(cuda_device)
    b = _train(cuda_device)
    assert a.keys() == b.keys()
    for k in a:
        assert a[k].shape == b[k].shape and torch.equal(a[k], b[k]), k
    assert a["_xyz"].shape[0] != 50000, "densify_and_prune changed nothing"


def test_image_loss_is_bit_identical_across_calls(cuda_device, det):
    from gaussianhaircut_b200 import losses as ghl
    W, H = 1920, 1080
    g = torch.Generator().manual_seed(3)
    r = lambda *s: torch.rand(*s, generator=g).to(cuda_device)  # noqa: E731
    render = torch.cat([r(3, H, W), r(2, H, W), r(3, H, W) * 2 - 1, r(1, H, W) * 0.9 + 0.05, r(1, H, W) * 3])
    gts = (r(3, H, W), (r(2, H, W) > 0.3).float(), r(1, H, W), r(1, H, W))
    ref = ghl.image_loss_forward_backward(render, *gts, 0.8, 0.2, 0.1, 0.1)
    for _ in range(5):
        l8, dL = ghl.image_loss_forward_backward(render, *gts, 0.8, 0.2, 0.1, 0.1)
        assert torch.equal(l8, ref[0]) and torch.equal(dL, ref[1])
