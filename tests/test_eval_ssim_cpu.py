"""CPU tests of the evaluation SSIM (gh_eval_ssim, inference.eval_ssim, evaluate_views(ssim=True), metrics.evaluate):
the float64 replay tests/_ssim64.py against the reference's own loss_utils.ssim and image_utils.psnr in float64 (live
where the reference sources are present, and through tests/golden/ssim64.npz everywhere); every refusal of the two C
entry points before any launch; evaluate_views' option handling and metrics.evaluate's directory walk and JSON layout
with the device calls stubbed."""
import ctypes as C
import json
import math
import os
import sys
import types

import numpy as np
import pytest
import torch

import _ssim64
import _util

sys.path.insert(0, os.path.join(_util.ROOT, "oracle"))
import ref_python  # noqa: E402

GOLDEN = os.path.join(_util.ROOT, "tests", "golden", "ssim64.npz")


@pytest.fixture(scope="module")
def lib():
    from gaussianhaircut_b200 import build, _capi
    build.build(verbose=False)
    return _capi.load()


# ------------------------------------------------------------------------------------------------ the float64 replay
def _assert_matches(ref):
    for name, (a, b, m) in _ssim64.cases().items():
        r = _ssim64.replay(a, b, m)
        s, p = ref[f"{name}/ssim"], ref[f"{name}/psnr"]
        assert abs(r["ssim"] - s) <= 1e-14, (name, r["ssim"], s)
        assert (r["psnr"] == p) if math.isinf(p) else abs(r["psnr"] - p) <= 1e-12 * abs(p), (name, r["psnr"], p)


def test_replay_matches_the_pinned_reference_outputs():
    with np.load(GOLDEN) as z:
        _assert_matches({k: float(z[k]) for k in z.files})


def test_replay_matches_the_reference_functions_live():
    if not ref_python.available():
        pytest.skip("reference Python sources not available")
    sys.path.insert(0, os.path.join(_util.ROOT, "tests", "golden"))
    import make_golden_ssim64
    ref = {}
    for name, (a, b, m) in _ssim64.cases().items():
        ref[f"{name}/ssim"], ref[f"{name}/psnr"] = make_golden_ssim64.reference_outputs(a, b, m)
    _assert_matches(ref)


def test_replay_cases_cover_the_edges():
    cases = _ssim64.cases()
    shapes = {a.shape[1:] for a, _, _ in cases.values()}
    assert {(1, 1), (5, 7), (10, 10), (11, 11), (17, 33), (64, 48)} <= shapes
    r = _ssim64.replay(*cases["const"])                      # sigma = 0: only C1 and C2 keep the ratio finite
    assert math.isfinite(r["ssim"]) and 0 < r["ssim"] < 1
    r = _ssim64.replay(*cases["identical"])
    assert r["ssim"] == 1.0 and r["psnr"] == math.inf and r["mse"] == 0.0
    a, b, _ = cases["render_bg"]
    assert np.mean(np.all(a == b, axis=0)) > 0.6               # mostly background
    # the cancellation in sigma = E[x^2] - mu^2 is what the bound of a flat image is made of
    assert _ssim64.replay(*cases["const"])["ssim_scale"] > 20 * _ssim64.replay(*cases["rand_64x48"])["ssim_scale"]


# ------------------------------------------------------------------------------------------------------ the C ABI
def test_entry_points_refuse_bad_arguments_without_a_device(lib):
    from gaussianhaircut_b200 import _capi
    E = _capi.GH_E_INVALID_ARG
    fake, n = C.c_void_p(0x1000), C.c_size_t()
    launches = lib.gh_kernel_launch_count()
    for B, W, H in ((0, 8, 8), (1, 0, 8), (1, 8, 0), (-1, 8, 8), (65536, 8, 8), (64, 8192, 8192)):
        assert lib.gh_eval_ssim_workspace_size(B, W, H, C.byref(n)) == E, (B, W, H)
        assert b"gh_eval_ssim_workspace_size" in lib.gh_last_error()
    assert lib.gh_eval_ssim_workspace_size(1, 8, 8, None) == E
    assert lib.gh_eval_ssim_workspace_size(3, 1920, 1080, C.byref(n)) == _capi.GH_OK and lib.gh_last_error() == b""
    tiles = ((1920 + 31) // 32) * ((1080 + 31) // 32)
    assert n.value == 8 * 3 * (4 + 2 * tiles)                  # per pair: 4 doubles of sums and ticket + 2 per CTA
    plane = 1920 * 1080

    def call(**kw):
        a = dict(B=3, W=1920, H=1080, img1=fake, d1=0, s1=3 * plane, img2=fake, d2=1, s2=3 * plane, mask=None, sm=0,
                 flags=0, ssim=fake, ss=8, psnr=None, sp=0, ws=fake, wsb=n.value, debug=0)
        a.update(kw)
        return lib.gh_eval_ssim(*a.values(), None)

    cases = {
        "bad B/width/height": [dict(B=0), dict(W=0), dict(H=-2)],
        "65535": [dict(B=65536)],
        "exceeds 2^31 - 1": [dict(B=400, s1=3 * plane, s2=3 * plane)],
        "unknown dtype": [dict(d1=2), dict(d2=-1)],
        "missing image": [dict(img1=None), dict(img2=None), dict(ssim=None), dict(ws=None)],
        "unknown flag": [dict(flags=8)],
        "overlap": [dict(s1=3 * plane - 1), dict(s2=10), dict(mask=fake, sm=plane - 1)],
        "beyond 2^31 - 1": [dict(s1=1 << 30)],
        "positive": [dict(ss=0), dict(psnr=fake, sp=-8)],
        "4-byte": [dict(img1=C.c_void_p(0x1002)), dict(ssim=C.c_void_p(0x1001)), dict(mask=C.c_void_p(0x1006), sm=plane)],
        "8-byte": [dict(ws=C.c_void_p(0x1004))],
        "needed": [dict(wsb=n.value - 8)],
    }
    for msg, kws in cases.items():
        for kw in kws:
            assert call(**kw) == E, (msg, kw)
            assert msg.encode() in lib.gh_last_error(), (msg, kw, lib.gh_last_error())
    assert call(img2=C.c_void_p(0x1003), d2=1, debug=0, ws=None) == E                # uint8 needs no alignment
    assert b"missing" in lib.gh_last_error()
    lib.gh_stage_timing_enable(1)
    try:
        assert call(debug=1) == E and b"stage timer" in lib.gh_last_error()
    finally:
        lib.gh_stage_timing_enable(0)
    assert lib.gh_kernel_launch_count() == launches


def test_eval_ssim_wrapper_refuses_cpu_tensors_and_bad_shapes():
    from gaussianhaircut_b200 import inference
    a = torch.zeros(3, 8, 8)
    with pytest.raises(RuntimeError, match="CUDA"):
        inference.eval_ssim(a, a, torch.zeros(1))
    with pytest.raises(RuntimeError, match="float32 or uint8"):
        inference.eval_ssim(a.double(), a, torch.zeros(1))


# -------------------------------------------------------------------------------------------- evaluate_views(ssim=)
class _StubRenderer:
    device = torch.device("cpu")
    capacity = 1

    def __init__(self):
        self.io = torch.zeros(2, dtype=torch.int32)

    def render_raw(self, view, check=True):
        return view.raw

    def after_readback(self, view, status, R, render=False):
        return False


def _stub_views(n=3, H=6, W=5):
    g = torch.Generator().manual_seed(3)
    views = []
    for k in range(n):
        v = types.SimpleNamespace(raw=torch.rand(10, H, W, generator=g), original_image=torch.rand(3, H, W, generator=g),
                                  original_mask=torch.rand(2, H, W, generator=g),
                                  original_orient_angle=torch.rand(1, H, W, generator=g),
                                  original_orient_conf=torch.rand(1, H, W, generator=g), k=k)
        views.append(v)
    return views


@pytest.fixture
def stubbed(monkeypatch):
    from gaussianhaircut_b200 import inference
    calls = {"metrics": [], "ssim": []}

    def eval_metrics(raw, gi, gm, ga, gc, stage, row, ws):
        calls["metrics"].append(stage)
        row.copy_(torch.arange(8, dtype=torch.float32) + float(raw[0, 0, 0]))
        row[4] = float("nan")

    def eval_ssim(img1, img2, out_ssim, out_psnr=None, clamp1=False, mask=None, workspace=None, clamp2=False,
                  clamp_mask=False, debug=False):
        calls["ssim"].append(dict(img1=img1, img2=img2, out=out_ssim, psnr=out_psnr, clamp1=clamp1, clamp2=clamp2,
                                  mask=mask, clamp_mask=clamp_mask, workspace=workspace))
        out_ssim.fill_(0.5 + float(img1[0, 0, 0]) / 10)

    monkeypatch.setattr(inference, "eval_metrics", eval_metrics)
    monkeypatch.setattr(inference, "eval_ssim", eval_ssim)
    monkeypatch.setattr(inference, "eval_workspace", lambda W, H, dev: torch.zeros(1, dtype=torch.float64))
    monkeypatch.setattr(inference, "ssim_workspace", lambda B, W, H, dev: torch.zeros(2, dtype=torch.float64))
    return calls


@pytest.mark.parametrize("stage", ["appearance", "strands", "latent_strands"])
def test_evaluate_views_ssim_option(stubbed, stage):
    from gaussianhaircut_b200 import inference
    views = _stub_views()
    plain = inference.evaluate_views(views, _StubRenderer(), stage)
    assert "ssim" not in plain and not stubbed["ssim"] and len(stubbed["metrics"]) == 3
    got = inference.evaluate_views(views, _StubRenderer(), stage, ssim=True)
    assert len(stubbed["ssim"]) == 3 and len(stubbed["metrics"]) == 6
    assert {k: v for k, v in got.items() if k != "ssim"} == plain      # the other slots are untouched
    want = np.mean([np.float32(0.5 + float(v.raw[0, 0, 0]) / 10) for v in views], dtype=np.float64)
    assert got["ssim"] == pytest.approx(want, rel=1e-6)
    for v, c in zip(views, stubbed["ssim"]):
        assert c["img1"].data_ptr() == v.raw.data_ptr() and tuple(c["img1"].shape) == (3, 6, 5)   # raw[:3], in place
        assert torch.equal(c["img2"], v.original_image) and c["clamp1"] and c["clamp2"] and c["psnr"] is None
        assert c["out"].numel() == 1 and c["workspace"] is not None
        if stage == "latent_strands":
            assert torch.equal(c["mask"], v.original_mask[:1]) and c["clamp_mask"]
        else:
            assert c["mask"] is None


def test_evaluate_views_ssim_argument(stubbed):
    from gaussianhaircut_b200 import inference
    for bad in ("yes", 1, None):
        with pytest.raises(TypeError, match="ssim"):
            inference.evaluate_views(_stub_views(), _StubRenderer(), "appearance", ssim=bad)
    assert inference.evaluate_views([], _StubRenderer(), "appearance", ssim=True) == {}
    assert not stubbed["metrics"] and not stubbed["ssim"]


# ------------------------------------------------------------------------------------------------ metrics.evaluate
def _png(path, a):
    from PIL import Image
    Image.fromarray(a).save(path)


def _tree(root, methods, rng, sizes=((12, 10),)):
    names = {}
    for m in methods:
        for d in ("renders", "gt"):
            os.makedirs(root / "test" / m / d)
        names[m] = []
        for i in range(5):
            H, W = sizes[i % len(sizes)]
            name = f"{i:05d}.png"
            ch = 4 if i == 1 else 3                                            # an RGBA render: [:, :3]
            _png(root / "test" / m / "renders" / name, rng.integers(0, 256, (H, W, ch), dtype=np.uint8))
            _png(root / "test" / m / "gt" / name, rng.integers(0, 256, (H, W, 3), dtype=np.uint8))
            names[m].append(name)
    return names


def _stub_ssim_psnr(renders, gts, device, chunk=16):
    s = torch.tensor([float(r.astype(np.float64).mean()) / 255 for r in renders], dtype=torch.float32)
    p = torch.tensor([float(g.astype(np.float64).mean()) / 10 for g in gts], dtype=torch.float32)
    return s, p


def test_metrics_evaluate_writes_the_reference_layout(tmp_path, monkeypatch, capsys):
    from gaussianhaircut_b200 import metrics
    monkeypatch.setattr(metrics, "ssim_psnr", _stub_ssim_psnr)
    rng = np.random.default_rng(4)
    scene = tmp_path / "scene"
    names = _tree(scene, ["ours_100", "ours_200"], rng, sizes=((12, 10), (7, 9)))
    full = metrics.evaluate([str(scene)], device="cpu")
    out = capsys.readouterr().out
    assert "LPIPS not computed" in out and out.count("LPIPS") == 1 and "Scene: " + str(scene) in out
    assert "  SSIM : " in out and "  PSNR : " in out
    res = json.load(open(scene / "results.json"))
    per = json.load(open(scene / "per_view.json"))
    assert full[str(scene)] == res
    assert set(res) == set(per) == {"ours_100", "ours_200"}
    for m in res:
        assert set(res[m]) == {"SSIM", "PSNR"} and set(per[m]) == {"SSIM", "PSNR"}
        assert set(per[m]["SSIM"]) == set(names[m])
        rs, gs, fn = metrics.read_images(scene / "test" / m / "renders", scene / "test" / m / "gt")
        s, p = _stub_ssim_psnr(rs, gs, "cpu")
        assert per[m]["SSIM"] == dict(zip(fn, s.tolist())) and per[m]["PSNR"] == dict(zip(fn, p.tolist()))
        assert res[m]["SSIM"] == s.mean().item() and res[m]["PSNR"] == p.mean().item()


def test_metrics_evaluate_with_lpips_fn_and_a_failing_scene(tmp_path, monkeypatch, capsys):
    from gaussianhaircut_b200 import metrics
    monkeypatch.setattr(metrics, "ssim_psnr", _stub_ssim_psnr)
    seen = []

    def lpips_fn(a, b):
        seen.append((tuple(a.shape), a.dtype, float(a.min()), float(a.max())))
        return torch.tensor([[[[float((a - b).abs().mean())]]]])

    scene = tmp_path / "scene"
    _tree(scene, ["ours_1"], np.random.default_rng(5))
    metrics.evaluate([str(tmp_path / "missing"), str(scene)], lpips_fn=lpips_fn, device="cpu")
    out = capsys.readouterr().out
    assert "Unable to compute metrics for model " + str(tmp_path / "missing") in out and "not computed" not in out
    res = json.load(open(scene / "results.json"))
    per = json.load(open(scene / "per_view.json"))
    assert set(res["ours_1"]) == {"SSIM", "PSNR", "LPIPS"} and len(per["ours_1"]["LPIPS"]) == 5
    assert len(seen) == 5 and all(s[0] == (1, 3, 12, 10) and s[1] == torch.float32 and 0 <= s[2] <= s[3] <= 1 for s in seen)


def test_metrics_reads_rgb_and_chunks_by_size(tmp_path):
    from gaussianhaircut_b200 import metrics
    a = np.random.default_rng(6).integers(0, 256, (4, 6, 4), dtype=np.uint8)
    _png(tmp_path / "a.png", a)
    got = metrics.read_png(tmp_path / "a.png")
    assert got.shape == (3, 4, 6) and got.dtype == np.uint8 and np.array_equal(got, a[:, :, :3].transpose(2, 0, 1))
    _png(tmp_path / "g.png", a[:, :, 0])
    with pytest.raises(RuntimeError, match="RGB"):
        metrics.read_png(tmp_path / "g.png")
    shapes = [np.zeros(s) for s in ((3, 4, 4),) * 5 + ((3, 2, 2),) * 2 + ((3, 4, 4),)]
    assert list(metrics._chunks(shapes, 2)) == [(0, 2), (2, 4), (4, 5), (5, 7), (7, 8)]
