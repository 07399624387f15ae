"""GPU tests of the evaluation SSIM (gh_eval_ssim, inference.eval_ssim, evaluate_views(ssim=True), metrics.evaluate):

  * every pair's SSIM and PSNR against the float64 replay tests/_ssim64.py, |kernel - replay| <= u * scale where scale
    is the replay's first-order bound of a float32 evaluation in the kernel's operation order (no calibrated
    constant), on the replay's cases (sizes 1x1 to 64x48, constant, identical, masked, background-heavy) and on 1080p
    and 2160p render-like pairs; the measured ratios are printed, and so is the difference of the reference's own
    loss_utils.ssim (staged under oracle/_ref/src) run in float32 with TF32 off;
  * batching: B = 1, 7, 64 with mixed content, pair i bit-identical alone and in the batch, and across two runs;
  * input forms: uint8 against torchvision's to_tensor of the same bytes bit for bit, the clamp against pre-clamped
    input, the mask against pre-multiplied input, strided views of raw (10,H,W) renders against contiguous copies;
  * evaluate_views(ssim=True) for the three stages on the render-maps test scenes: the other slots bit-identical to
    ssim=False, slot 4 equal to eval_ssim on each view's clamped raw image;
  * metrics.evaluate on a render set written by write_render_set plus a gt directory, against the replay.
"""
import json
import math
import os
import sys

import numpy as np
import pytest
import torch

import _ssim64
import _util

sys.path.insert(0, os.path.join(_util.ROOT, "oracle"))
import ref_python  # noqa: E402

pytestmark = pytest.mark.gpu
U = _ssim64.U


def _inf():
    from gaussianhaircut_b200 import inference
    return inference


def _run(a, b, dev, **kw):
    """eval_ssim on one pair or a batch -> (ssim, psnr) float32 numpy arrays."""
    a = torch.as_tensor(a).to(dev)
    b = torch.as_tensor(b).to(dev)
    B = 1 if a.dim() == 3 else a.shape[0]
    s = torch.full((B,), float("nan"), device=dev)
    p = torch.full((B,), float("nan"), device=dev)
    _inf().eval_ssim(a, b, s, p, **kw)
    return s.cpu().numpy(), p.cpu().numpy()


def _ratio(k, r, scale):
    if math.isinf(r) or math.isinf(k):
        assert k == r, (k, r)
        return 0.0
    return abs(k - r) / (U * scale)


def _check(name, k_ssim, k_psnr, r):
    rs, rp = _ratio(float(k_ssim), r["ssim"], r["ssim_scale"]), _ratio(float(k_psnr), r["psnr"], r["psnr_scale"])
    print(f"[ssim64] {name}: ssim {float(k_ssim):.9f} |d| {abs(float(k_ssim) - r['ssim']):.3e} ratio {rs:.3f}; "
          f"psnr {float(k_psnr):.6f} ratio {rp:.3f}")
    assert rs <= 1.0 and rp <= 1.0, (name, rs, rp)
    return rs, rp


def _ref_ssim():
    if not ref_python.available():
        return None
    sys.path.insert(0, ref_python.ref_src_dir())
    from utils.loss_utils import ssim
    return ssim


def _ref32(a, b, dev, mask=None):
    """The reference's own ssim in float32 on the GPU with TF32 off, or None where its sources are not staged."""
    ssim = _ref_ssim()
    if ssim is None:
        return None
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        x, y = torch.as_tensor(a).to(dev)[None], torch.as_tensor(b).to(dev)[None]
        if mask is not None:
            m = torch.as_tensor(mask).to(dev)[None]
            x, y = x * m, y * m
        with torch.no_grad():
            return float(ssim(x, y))
    finally:
        torch.backends.cudnn.allow_tf32 = prev


@pytest.mark.parametrize("name", list(_ssim64.cases()))
def test_pairs_against_the_float64_replay(cuda_device, name):
    a, b, m = _ssim64.cases()[name]
    kw = {} if m is None else {"mask": torch.from_numpy(m).to(cuda_device)}
    s, p = _run(a, b, cuda_device, **kw)
    r = _ssim64.replay(a, b, m, device=cuda_device)
    _check(name, s[0], p[0], r)
    ref = _ref32(a, b, cuda_device, m)
    if ref is not None:
        print(f"[ssim64] {name}: reference float32 (TF32 off) - replay = {ref - r['ssim']:+.3e}, "
              f"kernel - replay = {float(s[0]) - r['ssim']:+.3e}")


def _render_like(W, H, seed, dev):
    """A render and its ground truth at full size: smooth shading plus texture in an ellipse on a flat background."""
    g = torch.Generator(device=dev).manual_seed(seed)
    yy = torch.linspace(-1, 1, H, device=dev)[:, None]
    xx = torch.linspace(-1, 1, W, device=dev)[None, :]
    blob = ((yy / 0.7) ** 2 + (xx / 0.4) ** 2 < 1).float()
    shade = torch.stack([0.5 + 0.4 * torch.sin(3 * xx + k) * torch.cos(2 * yy) for k in range(3)])
    tex = torch.rand(3, H, W, generator=g, device=dev)
    bg = torch.tensor([0.05, 0.1, 0.2], device=dev)[:, None, None]
    ren = blob * (0.7 * shade + 0.3 * tex) + (1 - blob) * bg
    gt = blob * (0.7 * shade + 0.3 * (tex + 0.05 * torch.randn(3, H, W, generator=g, device=dev)).clamp(0, 1)) + (1 - blob) * bg
    return ren.float().contiguous(), gt.float().contiguous()


@pytest.mark.parametrize("W,H", [(1920, 1080), (3840, 2160)])
def test_full_size_against_the_float64_replay(cuda_device, W, H):
    a, b = _render_like(W, H, W, cuda_device)
    s, p = _run(a, b, cuda_device)
    r = _ssim64.replay(a, b, device=cuda_device)
    _check(f"{W}x{H}", s[0], p[0], r)
    ref = _ref32(a, b, cuda_device)
    if ref is not None:
        print(f"[ssim64] {W}x{H}: reference float32 (TF32 off) - replay = {ref - r['ssim']:+.3e}, "
              f"kernel - replay = {float(s[0]) - r['ssim']:+.3e}")
    del r
    torch.cuda.empty_cache()


def _mixed(B, H, W, dev, seed=0):
    g = torch.Generator(device=dev).manual_seed(seed)
    a = torch.rand(B, 3, H, W, generator=g, device=dev)
    b = (a + 0.2 * torch.randn(B, 3, H, W, generator=g, device=dev)).clamp(0, 1)
    for i in range(0, B, 5):
        b[i] = a[i]                                     # identical pairs: psnr inf
    for i in range(1, B, 5):
        a[i], b[i] = 0.25, 0.75                         # constant pairs
    for i in range(2, B, 5):
        b[i] = torch.rand(3, H, W, generator=g, device=dev)   # unrelated pairs
    return a.contiguous(), b.contiguous()


@pytest.mark.parametrize("B", [1, 7, 64])
def test_batch_is_independent_of_B_and_reproducible(cuda_device, B):
    a, b = _mixed(B, 45, 70, cuda_device, seed=B)
    s1, p1 = _run(a, b, cuda_device)
    s2, p2 = _run(a, b, cuda_device)
    assert np.array_equal(s1, s2) and np.array_equal(p1, p2)
    for i in range(B):
        si, pi = _run(a[i], b[i], cuda_device)
        assert s1[i].tobytes() == si[0].tobytes() and p1[i].tobytes() == pi[0].tobytes(), i
    for i in range(min(B, 7)):
        _check(f"B{B}[{i}]", s1[i], p1[i], _ssim64.replay(a[i], b[i], device=cuda_device))


def test_uint8_matches_to_tensor_bit_for_bit(cuda_device):
    import torchvision.transforms.functional as tf
    from PIL import Image
    g = np.random.default_rng(7)
    ua = g.integers(0, 256, (4, 37, 53, 3), dtype=np.uint8)
    ub = np.clip(ua.astype(np.int32) + g.integers(-20, 21, ua.shape), 0, 255).astype(np.uint8)
    ub[1] = ua[1]
    fa = torch.stack([tf.to_tensor(Image.fromarray(x)) for x in ua])
    fb = torch.stack([tf.to_tensor(Image.fromarray(x)) for x in ub])
    chw = lambda u: torch.from_numpy(np.ascontiguousarray(u.transpose(0, 3, 1, 2)))  # noqa: E731
    s8, p8 = _run(chw(ua), chw(ub), cuda_device)
    sf, pf = _run(fa, fb, cuda_device)
    sm, pm = _run(chw(ua), fb, cuda_device)                          # mixed dtypes
    assert s8.tobytes() == sf.tobytes() == sm.tobytes() and p8.tobytes() == pf.tobytes() == pm.tobytes()
    assert p8[1] == np.inf
    for i in range(4):
        _check(f"u8[{i}]", s8[i], p8[i], _ssim64.replay(fa[i], fb[i], device=cuda_device))


def test_clamp_and_mask_match_prepared_inputs(cuda_device):
    a, b, _ = _ssim64.cases()["outside01"]
    a, b = torch.from_numpy(a).to(cuda_device), torch.from_numpy(b).to(cuda_device) * 1.3 - 0.1
    on, pon = _run(a, b, cuda_device, clamp1=True, clamp2=True)
    pre, ppre = _run(a.clamp(0, 1), b.clamp(0, 1), cuda_device)
    assert on.tobytes() == pre.tobytes() and pon.tobytes() == ppre.tobytes()
    off, poff = _run(a, b, cuda_device)
    assert off[0] != on[0]
    _check("clamp off", off[0], poff[0], _ssim64.replay(a, b, device=cuda_device))
    _check("clamp on", on[0], pon[0], _ssim64.replay(a.clamp(0, 1), b.clamp(0, 1), device=cuda_device))
    one, _ = _run(a, b, cuda_device, clamp1=True)
    assert one[0] == _run(a.clamp(0, 1), b, cuda_device)[0][0]
    # mask: a batch of 3 with per-pair masks (one with values outside [0, 1] for clamp_mask)
    g = torch.Generator(device=cuda_device).manual_seed(9)
    A, Bm = _mixed(3, 33, 29, cuda_device, seed=9)
    M = torch.rand(3, 1, 33, 29, generator=g, device=cuda_device) * 1.4 - 0.2
    sm, pm = _run(A, Bm, cuda_device, mask=M)
    sp, pp = _run(A * M, Bm * M, cuda_device)
    assert sm.tobytes() == sp.tobytes() and pm.tobytes() == pp.tobytes()
    sc, _ = _run(A, Bm, cuda_device, mask=M, clamp_mask=True)
    Mc = M.clamp(0, 1)
    assert sc.tobytes() == _run(A * Mc, Bm * Mc, cuda_device)[0].tobytes()
    for i in range(3):
        _check(f"mask[{i}]", sm[i], pm[i], _ssim64.replay(A[i], Bm[i], M[i], device=cuda_device))


def test_strided_raw_images_are_read_in_place(cuda_device):
    g = torch.Generator(device=cuda_device).manual_seed(11)
    raw = torch.rand(5, 10, 41, 67, generator=g, device=cuda_device) * 1.2 - 0.1
    gt = torch.rand(5, 3, 41, 67, generator=g, device=cuda_device)
    s, p = _run(raw[:, :3], gt, cuda_device, clamp1=True)
    sc, pc = _run(raw[:, :3].contiguous(), gt, cuda_device, clamp1=True)
    assert s.tobytes() == sc.tobytes() and p.tobytes() == pc.tobytes()
    rows = torch.full((5, 8), -1.0, device=cuda_device)
    _inf().eval_ssim(raw[:, :3], gt, rows[:, 4], rows[:, 3], clamp1=True)
    r = rows.cpu().numpy()
    assert r[:, 4].tobytes() == s.tobytes() and r[:, 3].tobytes() == p.tobytes()
    assert np.all(np.delete(r, [3, 4], axis=1) == -1.0)                 # nothing else in the rows is written
    s0, _ = _run(raw[2, :3], gt[2], cuda_device, clamp1=True)           # a (10,H,W) view's raw[:3]
    assert s0[0] == s[2]


# ------------------------------------------------------------------------------------------------- evaluate_views
@pytest.mark.parametrize("stage,mode", [("appearance", "gaussians"), ("strands", "strands"), ("latent_strands", "segments")])
def test_evaluate_views_ssim(cuda_device, stage, mode):
    import test_gpu_render_maps as rm
    inference = _inf()
    args, kw, _ = rm._setup(mode, cuda_device)
    g = torch.Generator().manual_seed(23)
    views = []
    for k in (3, 9, 17, 33):
        v = rm._view(cuda_device, k)
        v.original_image = torch.rand(3, rm.H0, rm.W0, generator=g) * 1.1 - 0.05
        v.original_orient_angle = torch.rand(1, rm.H0, rm.W0, generator=g)
        v.original_mask = torch.rand(2, rm.H0, rm.W0, generator=g) * 1.2 - 0.1
        v.original_orient_conf = torch.rand(1, rm.H0, rm.W0, generator=g) * 3
        views.append(v)
    vr = inference.ViewRenderer(*args, **kw)
    plain = inference.evaluate_views(views, vr, stage)
    got = inference.evaluate_views(views, vr, stage, ssim=True)
    assert "ssim" not in plain and set(got) == set(plain) | {"ssim"}
    for k in plain:
        assert got[k] == plain[k] or (math.isnan(got[k]) and math.isnan(plain[k])), k
    per = []
    for v in views:
        raw = vr.render_raw(v).clone()
        gi, gm = v.original_image.to(cuda_device), v.original_mask.to(cuda_device)
        mask = gm[:1] if stage == "latent_strands" else None
        s, _ = _run(raw[:3], gi, cuda_device, clamp1=True, clamp2=True, mask=mask, clamp_mask=True)
        per.append(float(s[0]))
        m = None if mask is None else mask.clamp(0, 1)
        r = _ssim64.replay(raw[:3].clamp(0, 1), gi.clamp(0, 1), m, device=cuda_device)
        assert _ratio(float(s[0]), r["ssim"], r["ssim_scale"]) <= 1.0
    assert got["ssim"] == pytest.approx(float(np.mean(np.array(per, dtype=np.float32), dtype=np.float64)), rel=1e-12)
    assert 0.0 < got["ssim"] < 1.0


# ------------------------------------------------------------------------------------------------ metrics.evaluate
def test_metrics_evaluate_on_a_render_set(cuda_device, tmp_path):
    import torchvision.transforms.functional as tf
    from PIL import Image
    import test_gpu_render_maps as rm
    from gaussianhaircut_b200 import metrics
    inference = _inf()
    pc, bg = rm._gaussians(cuda_device), rm._bg(cuda_device)
    views = [rm._view(cuda_device, k, name=f"img_{k:04d}.png") for k in (3, 17, 40)]
    scene = tmp_path / "scene"
    root = inference.write_render_set(str(scene), "test", 7, views, inference.ViewRenderer(pc, rm.PIPE, bg))
    os.makedirs(os.path.join(root, "gt"))
    g = np.random.default_rng(12)
    for f in sorted(os.listdir(os.path.join(root, "renders"))):
        a = np.asarray(Image.open(os.path.join(root, "renders", f))).astype(np.int32)
        Image.fromarray(np.clip(a + g.integers(-12, 13, a.shape), 0, 255).astype(np.uint8)).save(os.path.join(root, "gt", f))
    for d in os.listdir(root):                                      # metrics walks renders and gt only
        if d not in ("renders", "gt"):
            os.rename(os.path.join(root, d), os.path.join(tmp_path, d))
    metrics.evaluate([str(scene)], device=cuda_device)
    per = json.load(open(scene / "per_view.json"))["ours_7"]
    res = json.load(open(scene / "results.json"))["ours_7"]
    assert set(res) == {"SSIM", "PSNR"} and len(per["SSIM"]) == 3
    for f, s in per["SSIM"].items():
        a = tf.to_tensor(Image.open(os.path.join(root, "renders", f)))[:3]
        b = tf.to_tensor(Image.open(os.path.join(root, "gt", f)))[:3]
        _check(f"metrics {f}", s, per["PSNR"][f], _ssim64.replay(a, b, device=cuda_device))
