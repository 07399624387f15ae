"""GPU tests of the inference side (gaussianhaircut_b200/inference.py, gh_render_maps, gh_eval_metrics):

  * ViewRenderer.render_raw is bit-identical to the raw image of renderer.render / render_hair_strands /
    render_hair_segments (and render_hair where the reference's model classes are staged), at a resolution that is not a
    multiple of 16, for a view that sees nothing, and across a capacity shortfall (one retry, same image);
  * gh_render_maps: the bytes of render and masks equal save_image's arithmetic in PyTorch on the same raw image, the
    float maps equal `_post`'s within 1e-6 (the angle) or exactly (the confidence), the orientation-derived bytes equal the float64 replay away from truncation
    boundaries and are never more than one level off, on rendered images and on a synthetic image holding the pixels
    the kernel branches on;
  * gh_eval_metrics against the float64 replay for the three stages, with the reference's NaN / inf for a zero weight
    sum and for identical images, bit-identical run to run;
  * write_render_set against the reference's render_set loop restated with renderer.render, vis_orient's formula and
    torchvision.utils.save_image; evaluate_views against training_report's loop body in PyTorch;
  * sweep returns each view's own maps and releases its pinned buffers; render_maps + gh_eval_metrics capture into a
    CUDA graph and replay to the same bytes.
"""
import gc
import math
import os
import sys
import types
import weakref

import numpy as np
import pytest
import torch

import _maps64
import _strands
import _util
from test_render_maps_cpu import _case

sys.path.insert(0, os.path.join(_util.ROOT, "oracle"))
import ref_python  # noqa: E402
import synth  # noqa: E402

pytestmark = pytest.mark.gpu
PIPE = types.SimpleNamespace(debug=False)
W0, H0 = 203, 131                     # not multiples of 16, W * H not a multiple of 4


def _bg(dev):
    return torch.tensor(synth.BG_DEFAULT, device=dev)


def _view(dev, k=3, W=W0, H=H0, away=False, name=None, device_tan=False, **kw):
    d = synth.make_camera(k, W, H, **kw)
    if away:                          # everything behind the near plane: R = 0
        wv = d["world_view_transform"].double()
        pm_t = torch.linalg.inv(wv) @ d["full_proj_transform"].double()
        wv[3, 2] -= 10.0
        d["world_view_transform"], d["full_proj_transform"] = wv.float().contiguous(), (wv @ pm_t).float().contiguous()
    v = ref_python.make_camera(d, dev)
    v.image_name = name or f"view_{k:03d}.png"
    if device_tan:
        v.tan_fov = torch.tensor([d["tanfovx"], d["tanfovy"]], dtype=torch.float32, device=dev)
    return v


def _gaussians(dev, P=20000, seed=1):
    s = synth.make_blob_scene(P, seed=seed, spread=0.1, max_scale=0.01)
    logit = lambda p: torch.log(p / (1 - p))  # noqa: E731
    t = lambda x: x.to(dev).contiguous()  # noqa: E731
    return types.SimpleNamespace(
        _xyz=t(s["xyz"]), _scaling=t(torch.log(s["scaling"])), _rotation=t(s["rotation"]), _features_dc=t(s["f_dc"]),
        _features_rest=t(s["f_rest"]), _opacity=t(logit(s["opacity"].clamp(1e-6, 1 - 1e-6))),
        _label=t(logit(s["label"].clamp(1e-6, 1 - 1e-6))), _orient_conf=t(torch.log(s["orient_conf"])), active_sh_degree=3)


def _head(dev, n_head=5000):
    h = synth.make_blob_scene(n_head, seed=2, spread=0.08, max_scale=0.004)
    g = torch.Generator().manual_seed(3)
    return types.SimpleNamespace(
        xyz_precomp=h["xyz"].to(dev), scaling_precomp=h["scaling"].to(dev),
        rotation_precomp=torch.nn.functional.normalize(h["rotation"], dim=1).to(dev),
        opacity_precomp=h["opacity"].reshape(-1, 1).to(dev), shs_view=(0.3 * torch.randn(n_head, 3, 16, generator=g)).to(dev))


def _strand_model(dev, S=300, L=33):
    poly = _strands.make_strand_polylines(S, L, seed=4)
    hair = types.SimpleNamespace(active_sh_degree=3, max_sh_degree=3, pts_origins=poly["origins"].to(dev),
                                 scale=poly["scale"] * torch.ones(1, device=dev))
    for n, k in (("_dirs", "dirs"), ("_features_dc", "f_dc"), ("_features_rest", "f_rest"), ("_orient_conf", "conf")):
        setattr(hair, n, poly[k].to(dev).contiguous())
    return hair


def _segment_model(dev, S=300, L=33):
    s = synth.make_strand_scene(S, seed=4, segments=L)
    t = lambda x: x.to(dev).contiguous()  # noqa: E731
    return types.SimpleNamespace(_xyz=t(s["xyz"]), _dir=t(s["dir"]), scale=2e-4 * torch.ones(1, device=dev),
                                 _features_dc=t(s["f_dc"]), _features_rest=t(s["f_rest"]),
                                 _orient_conf=t(torch.log(s["orient_conf"])), active_sh_degree=3)


def _setup(mode, dev):
    """(ViewRenderer arguments, the eager renderer.* call with the same inputs)"""
    from gaussianhaircut_b200 import renderer
    bg = _bg(dev)
    if mode == "gaussians":
        pc = _gaussians(dev)
        return (pc, PIPE, bg), {}, lambda v: renderer.render(v, pc, PIPE, bg)
    if mode == "hair":
        if not ref_python.available():
            pytest.skip("reference Python sources not staged (GaussianModelHair)")
        ref_python.load_renderer("mine")
        head = synth.make_blob_scene(5000, seed=2, spread=0.08, max_scale=0.004)
        pc, hair = ref_python.make_hair_models(head, synth.make_strand_scene(300, seed=4, segments=33), dev)
        return (pc, PIPE, bg), {"pc_hair": hair}, lambda v: renderer.render_hair(v, pc, hair, PIPE, bg)
    head = _head(dev)
    if mode == "strands":
        hair = _strand_model(dev)
        return (head, PIPE, bg), {"pc_hair": hair}, lambda v: renderer.render_hair_strands(v, head, hair, PIPE, bg)
    hair = _segment_model(dev)
    return (head, PIPE, bg), {"pc_hair": hair, "mode": "segments"}, lambda v: renderer.render_hair_segments(v, head, hair, PIPE, bg)


# ------------------------------------------------------------------------------------------------------- 1. render_raw
@pytest.mark.parametrize("mode", ["gaussians", "strands", "segments", "hair"])
def test_render_raw_is_bit_identical_to_the_training_forward(cuda_device, mode):
    from gaussianhaircut_b200 import inference
    args, kw, eager = _setup(mode, cuda_device)
    vr = inference.ViewRenderer(*args, **kw)
    assert vr.mode == mode
    empty, near, other = _view(cuda_device, 5, away=True), _view(cuda_device, 3), _view(cuda_device, 40, focal_factor=0.9)
    # a view that sees nothing: the background, and a capacity sized for R = 0 ...
    raw = vr.render_raw(empty)
    assert raw.requires_grad is False and raw.grad_fn is None
    assert torch.equal(raw, eager(empty)["raw"].detach())
    assert torch.equal(raw[:9], _bg(cuda_device)[:9, None, None].expand(9, H0, W0))
    retries = vr.retries
    # ... which the next view exceeds: one retry, the same image
    raw = vr.render_raw(near)
    want = eager(near)["raw"].detach()
    assert torch.equal(raw, want) and float(raw[3:5].sum()) > 0
    if mode != "hair":
        assert vr.retries == retries + 1 and vr.capacity >= vr.r_max > 256
    allocations = vr.allocations
    for v in (other, near, empty):
        assert torch.equal(vr.render_raw(v), eager(v)["raw"].detach())
    assert vr.allocations == allocations                   # one set of buffers for every view of this shape
    with torch.enable_grad():                               # no autograd node whatever the caller's mode
        assert vr.render_raw(near).grad_fn is None


# --------------------------------------------------------------------------------------------------- 2. gh_render_maps
def _torch_save_u8(x):
    return x.clone().mul(255).add_(0.5).clamp_(0, 255).to(torch.uint8)


def _check_maps(maps, raw):
    from gaussianhaircut_b200 import renderer
    H, W = raw.shape[1:]
    post = renderer._post(raw, torch.zeros(1, dtype=torch.int32, device=raw.device), None)
    assert torch.equal(maps["render_u8"], _torch_save_u8(raw[0:3]).permute(1, 2, 0))
    assert torch.equal(maps["hair_mask_u8"], _torch_save_u8(raw[3]))
    assert torch.equal(maps["head_mask_u8"], _torch_save_u8(raw[4]))
    assert torch.equal(maps["orient_conf_masked"], raw[8:9] * raw[3:4])
    # the kernel's angle is the image losses' device function; `_post` normalises through torch's norm kernel and clamps
    # at float32(0.999) instead of 1 - float32(1e-3), and acos amplifies both near the clamp: a few ulps of 1
    assert float((maps["orient_angle"] - post["orient_angle"]).abs().max()) <= 1e-6
    raw_np = raw.cpu().numpy()
    flips = {k: _maps64.check_bytes(maps[k].cpu().numpy(), raw_np, k) for k in ("orient_u8", "orient_vis_u8", "orient_conf_vis_u8")}
    for k in ("orient_angle", "orient_conf_masked"):
        assert maps[k].shape == (1, H, W)
    return flips


def test_render_maps_on_the_branch_pixels(cuda_device):
    from gaussianhaircut_b200 import inference
    raw = torch.from_numpy(_case()[0]).to(cuda_device)
    vr = inference.ViewRenderer(_gaussians(cuda_device, 64), PIPE, _bg(cuda_device))
    maps = vr.maps_of(raw)
    _check_maps(maps, raw)
    m32 = _maps64.render_maps(raw.cpu().numpy(), np.float32)
    # first row: zero direction (angle of the eps-normalised zero vector), dir.x == 0, the five axis angles
    assert np.max(np.abs(maps["orient_angle"].cpu().numpy()[0, 0, :11] - m32["orient_angle"][0, 0, :11])) <= 2e-7
    # a subset of the outputs leaves the others untouched
    before = {k: v.clone() for k, v in maps.items()}
    vr.maps_of(raw * 0.5, ("hair_mask_u8",))
    for k in before:
        assert torch.equal(vr._maps[k], before[k]) == (k != "hair_mask_u8"), k


@pytest.mark.parametrize("mode", ["gaussians", "strands"])
def test_render_maps_on_rendered_views(cuda_device, mode):
    from gaussianhaircut_b200 import inference
    args, kw, _ = _setup(mode, cuda_device)
    vr = inference.ViewRenderer(*args, **kw)
    for v in (_view(cuda_device, 3), _view(cuda_device, 20, W=512, H=384)):
        maps = vr.render_maps(v)
        print(mode, v.image_width, "bytes off by one near a boundary:", _check_maps(maps, vr._bufs["raw"]))


# -------------------------------------------------------------------------------------------------- 3. gh_eval_metrics
def _row(raw, gts, stage, dev):
    from gaussianhaircut_b200 import inference
    row = torch.full((8,), -1.0, device=dev)
    inference.eval_metrics(raw, *gts, stage, row)
    return row.cpu().numpy()


@pytest.mark.parametrize("stage", ["appearance", "strands", "latent_strands"])
def test_eval_metrics_match_the_float64_replay(cuda_device, stage):
    from gaussianhaircut_b200 import inference
    vr = inference.ViewRenderer(_gaussians(cuda_device), PIPE, _bg(cuda_device))
    code = inference.STAGES[stage]
    cases = [tuple(torch.from_numpy(a).to(cuda_device) for a in (_case()[0], *_case()[1]))]
    raw = vr.render_raw(_view(cuda_device, 3, W=512, H=384)).clone()
    g = torch.Generator().manual_seed(11)
    cases.append((raw, torch.rand(3, 384, 512, generator=g).to(cuda_device),
                  (torch.rand(2, 384, 512, generator=g) > 0.3).float().to(cuda_device),
                  torch.rand(1, 384, 512, generator=g).to(cuda_device), torch.rand(1, 384, 512, generator=g).to(cuda_device)))
    for raw, *gts in cases:
        got = _row(raw, gts, stage, cuda_device)
        want = _maps64.eval_metrics(raw.cpu().numpy(), *(t.cpu().numpy() for t in gts), code)
        # per-pixel float32 terms summed in double: the error scale is a few float32 ulps of each quantity
        np.testing.assert_allclose(got[[0, 1, 2, 3, 5, 6, 7]], want[[0, 1, 2, 3, 5, 6, 7]], rtol=2e-5, atol=1e-7)
        assert np.isnan(got[4])                                          # ssim: not computed
        assert np.array_equal(got, _row(raw, gts, stage, cuda_device), equal_nan=True)      # fixed summation order
    # zero weights: 0 / 0 = NaN like or_loss's sum / sum; identical images: mse 0 -> psnr inf like image_utils.psnr
    raw, gi, gm, ga, gc = cases[1]
    got = _row(raw, (gi, gm, ga, torch.zeros_like(gc)), stage, cuda_device)
    assert np.isnan(got[2]) and np.isfinite(got[[0, 1, 3]]).all()
    same = raw.clone()
    same[0:3] = gi.clamp(0, 1)
    got = _row(same, (gi, gm, ga, gc), stage, cuda_device)
    assert got[0] == 0 and np.isposinf(got[3]) and (got[5:8] == 0).all()


# ------------------------------------------------------------------------------------- 4. the scripts' loops, restated
def _vis_orient(orient_angle, mask):
    """src/utils/image_utils.py:22-37, in PyTorch as the reference runs it."""
    deg = orient_angle * 180
    tri = lambda c: torch.clamp(1 - torch.abs(deg - c) / 45., 0, 1)  # noqa: E731
    red, green, magenta, teal = tri(0.) + tri(180.), tri(90.), tri(45.), tri(135.)
    vec = lambda *c: torch.tensor(c)[:, None, None].to(deg.device)  # noqa: E731
    bgr = vec(0, 0, 1) * red + vec(0, 1, 0) * green + vec(1, 0, 1) * magenta + vec(1, 1, 0) * teal
    return torch.stack([bgr[2], bgr[1], bgr[0]], dim=0) * mask


def test_write_render_set_matches_the_render_set_loop(cuda_device, tmp_path):
    """src/render_gaussians.py:31-68 with renderer.render and torchvision.utils.save_image, against write_render_set."""
    import torchvision
    from PIL import Image
    from gaussianhaircut_b200 import inference, renderer
    pc, bg = _gaussians(cuda_device), _bg(cuda_device)
    views = [_view(cuda_device, k, name=f"img_{k:04d}.png") for k in (3, 17, 40)]
    ref_root = tmp_path / "ref" / "train_x" / "ours_7"
    for d in inference.RENDER_SET_MAPS:
        os.makedirs(ref_root / d)
    with torch.no_grad():
        for view in views:
            output = renderer.render(view, pc, PIPE, bg)
            hair_mask = output["mask"][:1]
            orient_conf = output["orient_conf"] * hair_mask
            images = {"renders": output["render"], "hair_masks": hair_mask, "head_masks": output["mask"][1:],
                      "orients": output["orient_angle"] * hair_mask, "orients_vis": _vis_orient(output["orient_angle"], hair_mask),
                      "orient_confs_vis": _vis_orient(output["orient_angle"], 1 - 1 / (orient_conf + 1))}
            base = os.path.basename(view.image_name).split('.')[0]
            for d, im in images.items():
                torchvision.utils.save_image(im, str(ref_root / d / (base + ".png")))
            torch.save(orient_conf, str(ref_root / "orient_confs" / (base + ".pth")))
    root = inference.write_render_set(str(tmp_path / "mine"), "train", 7, views, inference.ViewRenderer(pc, PIPE, bg), "_x")
    assert os.path.relpath(root, tmp_path / "mine") == os.path.join("train_x", "ours_7")
    tree = lambda r: sorted(os.path.relpath(os.path.join(p, f), r) for p, _, fs in os.walk(r) for f in fs)  # noqa: E731
    assert tree(root) == tree(ref_root) and len(tree(root)) == 21
    for rel in tree(root):
        if rel.endswith(".pth"):
            a, b = torch.load(os.path.join(root, rel)), torch.load(ref_root / rel)
            assert a.shape == b.shape == (1, H0, W0) and float((a - b.cpu()).abs().max()) <= 1e-6
            continue
        a, b = Image.open(os.path.join(root, rel)), Image.open(ref_root / rel)
        assert a.mode == b.mode == "RGB" and a.size == b.size
        diff = np.abs(np.asarray(a).astype(np.int32) - np.asarray(b).astype(np.int32))
        exact = rel.split(os.sep)[0] in ("renders", "hair_masks", "head_masks")
        assert diff.max() <= (0 if exact else 1), rel
        assert np.count_nonzero(diff) <= 1e-3 * diff.size, rel


def _training_report(views, render, stage):
    """The loop body of training_report (src/train_gaussians.py:252-281, src/train_latent_strands.py:233-262)."""
    l1 = lambda a, b: torch.abs(a - b).mean()  # noqa: E731
    psnr = lambda a, b: (20 * torch.log10(1.0 / torch.sqrt(((a - b) ** 2).view(a.shape[0], -1).mean(1, keepdim=True)))).mean()  # noqa: E731
    tot = np.zeros(4)
    for v in views:
        pkg = render(v)
        image, mask, ang = (torch.clamp(pkg[k], 0.0, 1.0) for k in ("render", "mask", "orient_angle"))
        gi, gm, ga = (torch.clamp(t.cuda(), 0.0, 1.0) for t in (v.original_image, v.original_mask, v.original_orient_angle))
        gc = v.original_orient_conf.cuda()
        d = ang - ga
        lo = torch.minimum(d.abs(), torch.minimum((d - 1).abs(), (d + 1).abs())) * math.pi * gm[:1]
        orient = (lo * gc).sum() / gc.sum()
        if stage == "latent_strands":
            terms = (l1(image * gm[:1], gi * gm[:1]),
                     torch.nn.functional.binary_cross_entropy(mask[:1].clamp(1e-3, 1.0 - 1e-3), gm[:1]), orient,
                     psnr(image * gm[:1], gi * gm[:1]))
        else:
            terms = (l1(image, gi), l1(mask, gm), orient, psnr(image, gi))
        tot += np.array([float(t.double()) for t in terms])
    return tot / len(views)


@pytest.mark.parametrize("stage", ["appearance", "latent_strands"])
def test_evaluate_views_matches_training_report(cuda_device, stage):
    from gaussianhaircut_b200 import inference
    args, kw, eager = _setup("gaussians" if stage == "appearance" else "segments", cuda_device)
    g = torch.Generator().manual_seed(21)
    views = []
    for k in (3, 9, 17, 33, 40):
        v = _view(cuda_device, k)
        v.original_image, v.original_orient_angle = torch.rand(3, H0, W0, generator=g), torch.rand(1, H0, W0, generator=g)
        v.original_mask = (torch.rand(2, H0, W0, generator=g) > 0.3).float()
        v.original_orient_conf = torch.rand(1, H0, W0, generator=g) * 3
        views.append(v)
    vr = inference.ViewRenderer(*args, **kw)
    got = inference.evaluate_views(views, vr, stage)
    with torch.no_grad():
        want = _training_report(views, eager, stage)
    keys = ("l1", "ce" if stage == "latent_strands" else "mask", "or", "psnr")
    assert set(got) == set(keys) | {"mse_r", "mse_g", "mse_b"}
    np.testing.assert_allclose([got[k] for k in keys], want, rtol=1e-5)
    assert got == inference.evaluate_views(views, vr, stage)              # capacity known: no retry, the same numbers


# ----------------------------------------------------------------------------------------------------------- 5. sweep
def test_sweep_returns_each_views_own_maps_and_releases_its_buffers(cuda_device):
    from gaussianhaircut_b200 import inference
    vr = inference.ViewRenderer(_gaussians(cuda_device), PIPE, _bg(cuda_device))
    views = [_view(cuda_device, k) for k in (3, 9, 17, 33, 40)]
    want = ("render_u8", "orient_vis_u8", "orient_conf_masked")
    expect = [{k: v.cpu().clone() for k, v in vr.render_maps(view, want).items()} for view in views]
    refs, seen = [], 0
    gen = inference.sweep(vr, views, want, depth=2)
    for i, (view, maps) in enumerate(gen):
        assert view is views[i]
        for k in want:
            assert maps[k].is_pinned() and torch.equal(maps[k], expect[i][k]), (i, k)
            refs.append(weakref.ref(maps[k]))
        seen += 1
        if i == 3:
            break
    assert seen == 4 and any(r() is not None for r in refs)
    gen.close()
    del maps
    gc.collect()
    assert all(r() is None for r in refs)                                 # closed early: the pinned buffers are gone
    assert [v for v, _ in inference.sweep(vr, views, want, depth=3)] == views


# ----------------------------------------------------------------------------------------------------- 6. CUDA graph
def test_render_maps_and_eval_metrics_capture_into_a_cuda_graph(cuda_device):
    from gaussianhaircut_b200 import inference
    vr = inference.ViewRenderer(_gaussians(cuda_device), PIPE, _bg(cuda_device))
    view = _view(cuda_device, 3, device_tan=True)
    g = torch.Generator().manual_seed(5)
    gts = (torch.rand(3, H0, W0, generator=g).to(cuda_device), (torch.rand(2, H0, W0, generator=g) > 0.3).float().to(cuda_device),
           torch.rand(1, H0, W0, generator=g).to(cuda_device), torch.rand(1, H0, W0, generator=g).to(cuda_device))
    row, ws = torch.zeros(8, device=cuda_device), inference.eval_workspace(W0, H0, cuda_device)
    for _ in range(2):                                                    # sizes the capacity, allocates every buffer
        maps = vr.render_maps(view)
        inference.eval_metrics(vr.render_raw(view, check=False), *gts, "appearance", row, ws)
    torch.cuda.synchronize()
    want = {k: v.clone() for k, v in maps.items()}
    want_row, allocations = row.clone(), vr.allocations
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = vr.render_maps(view, check=False)
        inference.eval_metrics(vr._bufs["raw"], *gts, "appearance", row, ws)
    assert vr.allocations == allocations
    for t in (*captured.values(), row):
        t.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert int(vr.io[0]) == 0
    for k in want:
        assert torch.equal(captured[k], want[k]), k
    assert torch.equal(row.view(torch.int32), want_row.view(torch.int32))
