"""CPU tests of the inference side (gaussianhaircut_b200/inference.py, gh_render_maps, gh_eval_metrics): the C ABI's
argument checks without a device; the numpy replay tests/_maps64.py against the reference's own vis_orient, psnr,
l1_loss, or_loss, ce_loss and save_image arithmetic (live where the reference sources are present, and through
tests/golden/mapsref.npz everywhere); maps_to_supervision against a PNG round trip through write_render_set's writer
and the loadCam recipe; sweep's buffer rotation with a stand-in renderer."""
import ctypes as C
import os
import sys
import types

import numpy as np
import pytest
import torch

import _maps64
import _util

sys.path.insert(0, os.path.join(_util.ROOT, "oracle"))
import ref_python  # noqa: E402

GOLDEN = os.path.join(_util.ROOT, "tests", "golden", "mapsref.npz")
H, W = 20, 26


def _case():
    """A seeded raw (10,H,W) image and ground truth maps with the pixels the kernels branch on in the first row:
    zero direction, dir.x == 0 (both signs of y), angles 0 / 45 / 90 / 135 / 180 degrees, masks exactly 0 and 1, and
    values outside [0, 1]."""
    g = np.random.default_rng(5)
    raw = g.uniform(-0.1, 1.1, (10, H, W)).astype(np.float32)
    raw[5:7] = g.normal(0, 1, (2, H, W)).astype(np.float32)
    raw[8] = np.exp(g.normal(0, 1, (H, W))).astype(np.float32)
    s = np.float32(np.sqrt(0.5))
    dirs = [(0, 0), (0, 1), (0, -1), (1, 1e-9), (s, s), (1, 0), (s, -s), (1e-9, -1), (-s, s), (-1, 0), (-s, -s)]
    for i, (x, y) in enumerate(dirs):
        raw[5, 0, i], raw[6, 0, i] = x, y
    raw[3, 0, :6], raw[3, 0, 6:12] = 0.0, 1.0
    raw[4, 1, :6], raw[4, 1, 6:12] = 1.0, 0.0
    gts = (g.uniform(-0.05, 1.05, (3, H, W)).astype(np.float32), (g.uniform(0, 1, (2, H, W)) > 0.4).astype(np.float32),
           g.uniform(0, 1, (1, H, W)).astype(np.float32), np.exp(g.normal(0, 1, (1, H, W))).astype(np.float32))
    return raw, gts


@pytest.fixture(scope="module")
def lib():
    from gaussianhaircut_b200 import build, _capi
    build.build(verbose=False)
    return _capi.load()


def test_entry_points_validate_their_arguments_without_a_device(lib):
    from gaussianhaircut_b200 import _capi
    fake, n = C.c_void_p(0x1000), C.c_size_t()
    launches = lib.gh_kernel_launch_count()
    outs = [None] * 8
    assert lib.gh_render_maps(0, 8, fake, *outs, None) == _capi.GH_E_INVALID_ARG and b"gh_render_maps" in lib.gh_last_error()
    assert lib.gh_render_maps(8, 8, None, *outs, None) == _capi.GH_E_INVALID_ARG and b"raw image" in lib.gh_last_error()
    assert lib.gh_render_maps(1 << 14, 1 << 14, fake, *outs, None) == _capi.GH_E_INVALID_ARG
    misaligned = [None, None, C.c_void_p(0x1002)] + [None] * 5
    assert lib.gh_render_maps(8, 8, fake, *misaligned, None) == _capi.GH_E_INVALID_ARG and b"aligned" in lib.gh_last_error()
    assert lib.gh_eval_metrics_workspace_size(0, 8, C.byref(n)) == _capi.GH_E_INVALID_ARG
    assert lib.gh_eval_metrics_workspace_size(1920, 1080, C.byref(n)) == _capi.GH_OK and lib.gh_last_error() == b""
    # 16 doubles of sums and ticket + 7 sums per CTA
    ctas = min((1920 * 1080 + 255) // 256, 132 * 16)
    assert n.value == 8 * (16 + 7 * ctas)
    ok = (fake, fake, fake, fake, fake, fake, n.value, fake, None)
    assert lib.gh_eval_metrics(1920, 0, 0, *ok) == _capi.GH_E_INVALID_ARG
    assert lib.gh_eval_metrics(1920, 1080, 3, *ok) == _capi.GH_E_INVALID_ARG and b"stage" in lib.gh_last_error()
    assert lib.gh_eval_metrics(1920, 1080, 0, None, *ok[1:]) == _capi.GH_E_INVALID_ARG
    small = ok[:6] + (n.value - 8,) + ok[7:]
    assert lib.gh_eval_metrics(1920, 1080, 0, *small) == _capi.GH_E_INVALID_ARG and b"needed" in lib.gh_last_error()
    odd = ok[:5] + (C.c_void_p(0x1004),) + ok[6:]
    assert lib.gh_eval_metrics(1920, 1080, 0, *odd) == _capi.GH_E_INVALID_ARG and b"8-byte" in lib.gh_last_error()
    assert lib.gh_kernel_launch_count() == launches


def _assert_matches_reference(ref):
    raw, gts = _case()
    m32 = _maps64.render_maps(raw, np.float32)
    # bytes whose only float input is the raw image: the float32 replay is save_image's arithmetic exactly
    assert np.array_equal(m32["render_u8"], ref["render_u8"]) and np.array_equal(m32["hair_mask_u8"], ref["hair_mask_u8"])
    assert np.max(np.abs(m32["orient_angle"] - ref["orient_angle"])) <= 2 * np.finfo(np.float32).eps
    assert np.max(np.abs(_maps64.orient_angle(raw) - ref["orient_angle"])) <= 4e-6      # acos near +-0.999 amplifies
    for k in ("orient_u8", "orient_vis_u8", "orient_conf_vis_u8"):
        _maps64.check_bytes(ref[k], raw, k)
        _maps64.check_bytes(m32[k], raw, k)
    for stage, key in ((0, "row_stage0"), (2, "row_stage2")):
        row = _maps64.eval_metrics(raw, *gts, stage)
        np.testing.assert_allclose(row[:4], ref[key], rtol=2e-5)


def test_replay_matches_the_pinned_reference_outputs():
    with np.load(GOLDEN) as z:
        _assert_matches_reference({k: z[k] for k in z.files})


def test_replay_matches_the_reference_functions_live():
    if not ref_python.available():
        pytest.skip("reference Python sources not available")
    sys.path.insert(0, os.path.join(_util.ROOT, "tests", "golden"))
    import make_golden_maps
    _assert_matches_reference(make_golden_maps.reference_outputs(*_case()))


def test_float32_replay_quantises_like_save_image():
    """save_image's bytes are x.mul(255).add_(0.5).clamp_(0, 255).to(uint8): two rounded float32 operations, then
    truncation; the float32 replay -- and the kernel, tests/test_gpu_render_maps.py -- reproduce them for every x."""
    x = torch.cat([torch.linspace(-0.01, 1.01, 1 << 20), (torch.arange(256) + 0.5) / 255, torch.arange(256) / 255.0])
    two = x.clone().mul(255).add_(0.5).clamp_(0, 255).to(torch.uint8).numpy()
    assert np.array_equal(_maps64.quant(x.numpy(), np.float32), two)


def test_maps_to_supervision_equals_the_png_round_trip(tmp_path):
    """write_render_set's PNG writer + loadCam's reader (camera_utils.py:51-78, PILtoTorch at the stored resolution)."""
    from PIL import Image
    from gaussianhaircut_b200 import inference
    raw, _ = _case()
    maps = {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in _maps64.render_maps(raw, np.float32).items()}
    maps["orient_conf_masked"] = maps["orient_conf_masked"].float()
    load = {}
    for d, k in inference.RENDER_SET_MAPS.items():
        path = str(tmp_path / (d + (".pth" if k == "orient_conf_masked" else ".png")))
        if k == "orient_conf_masked":
            torch.save(maps[k].clone(), path)
            load[k] = torch.nn.functional.interpolate(torch.load(path).float()[None], size=(H, W), mode="bilinear")[0]
        else:
            inference.save_png(maps[k], path)
            img = Image.open(path)
            assert img.mode == "RGB" and img.size == (W, H)
            t = torch.from_numpy(np.array(img.resize((W, H)))) / 255.0             # PILtoTorch
            load[k] = t.permute(2, 0, 1)
    for binarize in (False, True):
        sup = inference.maps_to_supervision(maps, binarize_masks=binarize)
        hair, body = load["hair_mask_u8"][:1], load["head_mask_u8"][:1]
        if binarize:
            hair, body = (hair >= 0.5).float(), (body >= 0.5).float()
        want = {"image": load["render_u8"][:3], "mask_hair": hair, "mask_body": body,
                "orient_angle": load["orient_u8"][:1], "orient_conf": load["orient_conf_masked"][:1]}
        assert set(sup) == set(want)
        for k in want:
            assert sup[k].dtype == torch.float32 and torch.equal(sup[k], want[k]), k


class _StandIn:
    """render_maps of view i fills the one device-side buffer set with i, like ViewRenderer overwrites its maps."""
    device = torch.device("cpu")

    def __init__(self, overflow_on=()):
        self.io = torch.zeros(2, dtype=torch.int32)
        self.capacity, self.calls, self.overflow_on = 1, [], set(overflow_on)
        self._maps = {"render_u8": torch.zeros(2, 3, 3, dtype=torch.uint8), "orient_angle": torch.zeros(1, 2, 3)}

    def render_maps(self, view, want, check=True):
        self.calls.append((view, check))
        over = view in self.overflow_on and not check
        self.io[0], self.io[1] = int(over), 100 + view
        for k in want:
            self._maps[k].fill_(255 if over else view)
        return {k: self._maps[k] for k in want}

    def after_readback(self, view, status, R, render=False):
        assert R == 100 + view
        if status & 1:
            self.overflow_on.discard(view)
        return bool(status & 1)


@pytest.mark.parametrize("depth", [2, 3])
def test_sweep_yields_each_views_own_maps_one_behind(depth):
    from gaussianhaircut_b200 import inference
    r = _StandIn(overflow_on={2})
    want = ("render_u8", "orient_angle")
    seen, held = [], []
    for view, maps in inference.sweep(r, range(5), want, depth=depth):
        assert len(r.calls) - (2 in [v for v, c in r.calls if c]) == min(view + 2, 5)      # one view ahead of the caller
        assert set(maps) == set(want)
        assert int(maps["render_u8"][0, 0, 0]) == view and float(maps["orient_angle"][0, 0, 0]) == float(view)
        seen.append(view)
        held.append(maps["render_u8"])
        for back, t in enumerate(reversed(held[-(depth - 1):])):        # valid until depth - 1 further items
            assert int(t[0, 0, 0]) == view - back
    assert seen == list(range(5))
    assert (2, True) in r.calls                                          # the overflowed view was rendered again
    assert len({t.data_ptr() for t in held}) == depth                   # `depth` rotating buffer sets


def test_sweep_rejects_a_single_buffer_and_unknown_maps():
    from gaussianhaircut_b200 import inference
    with pytest.raises(RuntimeError, match="depth"):
        next(inference.sweep(_StandIn(), range(3), ("render_u8",), depth=1))
    with pytest.raises(RuntimeError, match="unknown map"):
        next(inference.sweep(_StandIn(), range(3), ("depth_u8",)))
