"""GPU tests: gh_image_loss element by element against the float64 replay (oracle/loss64.py), on the default and on
the deterministic path (torch.use_deterministic_algorithms(True), set by a local fixture).

Each case checks:
  * every dL/dout element: |k - r| <= TOL * scale, and exactly 0 where the replay's scale is 0 (channels 7 and 9,
    channels 0..2 where gt_mask[1] = 0, the orientation channels at exact ties and clamps, everything the NaN guard
    zeroes);
  * every loss value within TOL of its own scale, and the NaN flag exactly;
  * at pixels whose orientation decisions lie within float32 error of their thresholds (the replay's ratios below
    DECISION_SAFETY), any of the gradients the ambiguous decisions can give; such pixels are counted: none on the
    constructed scenes, at most AMBIGUOUS_MAX of the pixels on random ones.

Cases: sizes around the 11-tap window and the 32x32 tile, a real render with background pixels, exact ties, the NaN
guard through one pixel, CTA counts around the deterministic sums' 256-slot chunks and caps, the 2^27-pixel limit on
sampled windows, and the Python wrapper's dtype and layout conversions.

TOL was calibrated with tools/loss_replay_calibrate.py: the float32 restatement (oracle/loss_oracle.py on the CPU and
on the GPU with TF32 off) and this build through the same checks on the same scenes; TOL leaves the restatement's worst
ratio a factor of at least 4.
"""
import math
import os
import sys
import types

import numpy as np
import pytest
import torch

import _util

sys.path.insert(0, os.path.join(_util.ROOT, "oracle"))
import loss64  # noqa: E402
import synth  # noqa: E402

pytestmark = pytest.mark.gpu

# Calibrated on an H100 80GB HBM3 at a 400 W power limit (tools/loss_replay_calibrate.py; DESIGN.md, row 4).
# The float32 restatement's worst ratio is 7.9e-8 (CPU 5.9e-8), this build's 3.7e-8; TOL leaves the restatement 5x.
TOL = 4e-7
# Ambiguous pixels of a random scene: 18 and 33 of 2073600 on the two 1080p edge scenes (1.6e-5), so the bound is
# 2e-5 of the pixels, with a floor of AMBIGUOUS_FLOOR pixels for small scenes.
AMBIGUOUS_MAX = 2e-5
AMBIGUOUS_FLOOR = 8
LAMBDAS = (0.8, 0.2, 0.4, 0.1)


@pytest.fixture(params=[False, True], ids=["default", "deterministic"])
def det(request):
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(request.param)
    yield request.param
    torch.use_deterministic_algorithms(prev, warn_only=warn)


def _ghl():
    from gaussianhaircut_b200 import losses
    return losses


def compare(losses, dL, r, nan_flag=None, origin=(0, 0)):
    """The checks of the module docstring for one result (losses may be None for a crop).  Returns the worst ratios
    {name: ratio} and the number of ambiguous pixels; raises on any element the replay calls exact that is not."""
    dev = r["dL"].device
    k = dL.to(dev).double()
    assert bool(torch.isfinite(k).all()), "non-finite gradient"
    s = r["scale"]
    d = (k - r["dL"]).abs()
    y0, x0 = origin
    amb = torch.zeros_like(d, dtype=torch.bool)
    for (y, x) in r["alternatives"]:
        amb[5:7, y - y0, x - x0] = True                # checked against the alternatives below
    bad = (s == 0) & (d != 0) & ~amb
    assert not bool(bad.any()), f"{int(bad.sum())} elements must be exactly {0} (first at {torch.nonzero(bad)[0].tolist()})"
    ratio = torch.where(s > 0, d / s.clamp(min=1e-300), torch.zeros_like(d))
    amb_worst = 0.0
    def off(kv, a, e):
        return abs(kv - a) / e if e > 0 else (0.0 if kv == a else math.inf)
    for (y, x), (names, vals) in r["alternatives"].items():
        ly, lx = y - y0, x - x0
        k5, k6 = float(k[5, ly, lx]), float(k[6, ly, lx])
        amb_worst = max(amb_worst, min(max(off(k5, a5, e5), off(k6, a6, e6)) for a5, a6, e5, e6 in vals))
        ratio[5:7, ly, lx] = 0.0
    worst = {f"ch{c}": float(ratio[c].max()) for c in range(10)}
    worst["ambiguous"] = amb_worst
    if losses is not None:
        lv = losses.double().cpu()
        for i, n in enumerate(loss64.LOSSES):
            worst[n] = abs(float(lv[i]) - r["losses"][n]) / r["losses_scale"][n] if r["losses_scale"][n] else (
                0.0 if float(lv[i]) == r["losses"][n] else math.inf)
        flag = bool(lv[6] == 1.0) if nan_flag is None else nan_flag
        assert flag == r["nan"], f"NaN flag {flag}, replay {r['nan']}"
    return worst, len(r["alternatives"])


def assert_within(worst, n_amb, n_pixels, constructed=False):
    bad = {k: v for k, v in worst.items() if not v <= TOL}
    assert not bad, f"beyond {TOL} of the replay's scale: {bad}"
    if constructed:
        assert n_amb == 0, f"{n_amb} pixels at an ambiguous decision on a constructed scene"
    else:
        assert n_amb <= max(AMBIGUOUS_FLOOR, AMBIGUOUS_MAX * n_pixels), f"{n_amb} ambiguous pixels of {n_pixels}"


def run_check(ins, device, ws=None, lambdas=LAMBDAS):
    t = [x.to(device) for x in ins]
    losses, dL = _ghl().image_loss_forward_backward(*t, *lambdas, workspace=ws)
    r = loss64.replay(*t, lambdas, device=device)
    return (losses, dL, r) + compare(losses, dL, r)


# ------------------------------------------------------------------------------------------------- scenes
SIZES = [(1, 1), (1, 37), (37, 1), (5, 7), (10, 11), (11, 10), (31, 33), (32, 32), (33, 31), (63, 65), (4099, 3),
         (3, 4099), (250, 187), (1920, 1080)]


def real_render(device, W, H, seed=0):
    """renderer.render_raw of a synth strand scene over BG_DEFAULT (zero in channels 5..8), binary gt_mask, with
    zero-direction pixels that have conf > 0 and directions of norm 1e-13, 1e-12 and 2e-12 placed on the background."""
    sys.path.insert(0, os.path.join(_util.ROOT, "oracle"))
    import ref_python
    from gaussianhaircut_b200 import renderer
    scene = synth.make_strand_scene(300, seed=seed)
    raw = synth.raw_params_from_scene(scene, "gaussian_model")
    names = ("_xyz", "_features_dc", "_features_rest", "_opacity", "_label", "_scaling", "_rotation", "_orient_conf")
    keys = ("xyz", "f_dc", "f_rest", "opacity", "label", "scaling", "rotation", "conf")
    pc = types.SimpleNamespace(active_sh_degree=3, max_sh_degree=3)
    for n, k in zip(names, keys):
        setattr(pc, n, torch.nn.Parameter(raw[k].to(device).contiguous()))
    cam = ref_python.make_camera(synth.make_camera(0, W, H), device)
    bg = torch.tensor(synth.BG_DEFAULT, device=device)
    with torch.no_grad():
        out = renderer.render_raw(cam, pc, types.SimpleNamespace(debug=False), bg)[0].detach().float().contiguous()
    g = torch.Generator().manual_seed(seed + 1)
    r = lambda *s: torch.rand(*s, generator=g).to(device)   # noqa: E731
    gi, gm, ga, gc = r(3, H, W), (r(2, H, W) > 0.4).float(), r(1, H, W), r(1, H, W)
    bgpix = torch.nonzero((out[5:9] == 0).all(0))
    n_bg = bgpix.shape[0]
    pick = bgpix[torch.randperm(n_bg, generator=g)[:40].to(device)]
    vals = [(0.0, 0.0)] * 16 + [(0.6e-13, 0.8e-13)] * 8 + [(1e-12, 0.0), (0.0, 1e-12), (-1e-12, 0.0)] * 3 + \
        [(1.2e-12, -1.6e-12), (-2e-12, 0.0)] * 3
    for (y, x), (c5, c6) in zip(pick.tolist(), vals):
        out[5, y, x], out[6, y, x], out[8, y, x] = c5, c6, 0.7
        gm[0, y, x], gc[0, y, x] = 1.0, 0.5
    return (out, gi, gm, ga, gc), n_bg


# ------------------------------------------------------------------------------------------------- tests
@pytest.mark.parametrize("W,H", SIZES, ids=[f"{w}x{h}" for w, h in SIZES])
def test_sizes(cuda_device, det, W, H):
    ins = loss64.edge_scene(W, H, seed=W * 7 + H)
    *_, worst, n_amb = run_check(ins, cuda_device)
    print(f"{W}x{H} det={det}: worst {max(worst.values()):.3g}, ambiguous {n_amb}")
    assert_within(worst, n_amb, W * H)


@pytest.mark.parametrize("W,H", [(512, 384), (1920, 1080)])
def test_real_render(cuda_device, det, W, H):
    ins, n_bg = real_render(cuda_device, W, H)
    out, gm, gc = ins[0], ins[2], ins[4]
    bg = (out[5:9] == 0).all(0)
    assert n_bg > W * H // 10 and bool((bg & (gm[0] == 1) & (gc[0] > 0)).any()), "no supervised background pixels"
    losses, dL, r, worst, n_amb = run_check(ins, cuda_device)
    eps_px = (out[8] > 0) & (out[5] == 0) & (out[6] == 0)
    assert int(eps_px.sum()) >= 16 and float(r["dL"][6][eps_px].abs().min()) > 1e3, "the eps gradient is not reached"
    print(f"render {W}x{H} det={det}: worst {max(worst.values()):.3g}, ambiguous {n_amb}")
    assert_within(worst, n_amb, W * H)


def test_exact_ties(cuda_device, det):
    """ang = acos(0) / pi = 0.5 exactly (asserted on the device), with gt_angle 0, 0.5, 1: the torch.minimum tie,
    d0 = 0 and l0 = l2; clamps at |c6| = 1; (3, 4); image and mask equalities; a masked-out block larger than the
    window and a constant block.  Every decision is exact: no ambiguous pixel."""
    z = torch.zeros(4, device=cuda_device)
    assert bool((torch.acos(z) / math.pi == 0.5).all()), "acos(0) / pi is not 0.5 on this device: the tie is not reached"
    ins = loss64.edge_scene(48, 40, seed=5)
    losses, dL, r, worst, n_amb = run_check(ins, cuda_device)
    out = ins[0]
    ties = (out[6] == 0) & (out[5].abs() == 1)
    assert int(ties.sum()) == 6 and bool((r["scale"][5:7][:, ties.to(cuda_device)] == 0).all())
    assert bool((r["scale"][0:3, 2:15, 3:16] == 0).all())                      # the masked-out block
    assert_within(worst, n_amb, 48 * 40, constructed=True)


def test_nan_guard_through_a_pixel(cuda_device, det):
    ins = list(loss64.edge_scene(64, 48, seed=8, specials=False))
    ins[0][8, 17, 23] = -float(np.float32(1e-7))
    ins[2][0, 17, 23] = 0.0
    losses, dL, r, worst, n_amb = run_check(ins, cuda_device)
    assert r["nan"] and float(losses[6]) == 1.0 and float(losses[4]) == 0.0
    assert not bool(dL[[5, 6, 8]].any()), "the NaN guard left an orientation gradient"
    assert_within(worst, n_amb, 64 * 48, constructed=True)


# (W, H): presum / pointwise CTAs ceil(W H / 256) up to the caps 1056 / 2112, SSIM CTAs = 32x32 tiles
DET_SHAPES = {
    "cta255": (255, 256), "cta256": (256, 256), "cta257": (257, 256),        # presum = pointwise = 255, 256, 257
    "cta600": (480, 320),                                                    # 3 chunks, last one partial
    "tiles255": (480, 544), "tiles256": (512, 512), "tiles257": (8219, 30),  # SSIM CTAs 15x17, 16x16, 257x1
    "plane270337": (270337, 1),                                              # presum cap 1056 * 256 + 1
    "plane540673": (77239, 7),                                               # pointwise cap 2112 * 256 + 1
    "1080p": (1920, 1080),                                                   # 2040 tiles: 8 chunks
}


@pytest.mark.parametrize("name", list(DET_SHAPES))
def test_deterministic_sums(cuda_device, det, name):
    W, H = DET_SHAPES[name]
    ghl = _ghl()
    ws = torch.empty(ghl.workspace_elems(2048, 1100), dtype=torch.float64, device=cuda_device)
    big = [t.to(cuda_device) for t in loss64.edge_scene(2048, 1100, seed=99, specials=False)]
    ghl.image_loss_forward_backward(*big, *LAMBDAS, workspace=ws)          # leaves ws dirty
    ins = loss64.edge_scene(W, H, seed=W + H)
    losses, dL, r, worst, n_amb = run_check(ins, cuda_device, ws=ws)
    assert_within(worst, n_amb, W * H)
    if det:
        t = [x.to(cuda_device) for x in ins]
        l2, d2 = ghl.image_loss_forward_backward(*t, *LAMBDAS, workspace=ws)
        assert torch.equal(l2, losses) and torch.equal(d2, dL), "not bit-identical across calls"


def test_size_limit(cuda_device, det):
    """W H = 2^27 (16384 x 8192): the sums against float64 sums formed in bands, dL on crops (the four corners, the
    last row and column, 64 random windows)."""
    W, H = 16384, 8192
    free = torch.cuda.mem_get_info(cuda_device)[0]
    if free < 24 * 2 ** 30:
        pytest.skip(f"needs 24 GiB free, the device has {free / 2 ** 30:.1f} GiB")
    g = torch.Generator(device=cuda_device).manual_seed(5)
    r = lambda *s: torch.rand(*s, generator=g, device=cuda_device)   # noqa: E731
    out = torch.empty(10, H, W, device=cuda_device)
    out[0:5] = r(5, H, W)
    out[5:8] = r(3, H, W) * 2 - 1
    out[8] = r(H, W) * 0.9 + 0.05
    out[9] = 0
    ins = [out, r(3, H, W), (r(2, H, W) > 0.3).float(), r(1, H, W), r(1, H, W)]
    losses, dL = _ghl().image_loss_forward_backward(*ins, *LAMBDAS)
    s = loss64.chunked_sums(ins, LAMBDAS, rows=128, device=cuda_device)
    lv = losses.double().cpu()
    for i, n in enumerate(loss64.LOSSES):
        assert abs(float(lv[i]) - s["losses"][n]) <= TOL * s["losses_scale"][n], n
    assert bool(lv[6] == 0.0) and not s["nan"]
    sw = (s["sums"]["w"], s["sums_scale"]["w"])
    rng = np.random.default_rng(0)
    rects = [(0, 0, 48, 48), (W - 48, 0, W, 48), (0, H - 48, 48, H), (W - 48, H - 48, W, H),
             (0, H - 1, W, H), (W - 1, 0, W, H)]
    for _ in range(64):
        x, y = int(rng.integers(0, W - 32)), int(rng.integers(0, H - 32))
        rects.append((x, y, x + 32, y + 32))
    n_amb, n_px = 0, 0
    for x0, y0, x1, y1 in rects:
        c = loss64.replay_crop(ins, LAMBDAS, x0, y0, x1, y1, sw, device=cuda_device)
        worst, na = compare(None, dL[:, y0:y1, x0:x1], c, origin=c["origin"])
        bad = {k: v for k, v in worst.items() if not v <= TOL}
        assert not bad, f"crop {(x0, y0, x1, y1)}: {bad}"
        n_amb, n_px = n_amb + na, n_px + (x1 - x0) * (y1 - y0)
    print(f"2^27 case ran (det={det}): {n_px} pixels checked, ambiguous {n_amb}")
    assert n_amb <= max(AMBIGUOUS_FLOOR, AMBIGUOUS_MAX * n_px)


def test_wrapper_conversions_are_exact(cuda_device):
    """float16 / uint8 / bool maps and non-contiguous views give the bits of their float32 contiguous copies."""
    ghl = _ghl()
    W, H = 70, 45
    out, gi, gm, ga, gc = (t.to(cuda_device) for t in loss64.edge_scene(W, H, seed=12))
    gm_b = gm > 0.5
    stack = torch.cat([gm_b[:1].float(), gm_b.float()])                     # gt_mask[1:] of a 3-channel map
    hwc = out.permute(1, 2, 0).contiguous().permute(2, 0, 1)               # a permuted HWC render
    gi_h = gi.half()
    ga_u8 = (ga * 255).to(torch.uint8)
    gc_hwc = gc.permute(1, 2, 0).contiguous().permute(2, 0, 1)
    views = [(hwc, gi_h, gm_b, ga_u8, gc_hwc), (out, gi_h.permute(0, 2, 1).contiguous().permute(0, 2, 1), stack[1:],
                                               ga_u8.float(), gc[:, :, :]),
             (out[:, :, :], gi, gm_b.to(torch.uint8), ga, gc.half())]
    assert not hwc.is_contiguous() and not views[1][1].is_contiguous()
    for v in views:
        ref = [t.float().contiguous() for t in v]
        a = ghl.image_loss_forward_backward(*v, *LAMBDAS)
        b = ghl.image_loss_forward_backward(*ref, *LAMBDAS)
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
