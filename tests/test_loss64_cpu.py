"""CPU tests: pin the float64 loss replay (oracle/loss64.py) on the reference's own loss functions run in float64
(tests/golden/loss64edges.npz, tests/golden/make_golden_loss64.py) and on float64 autograd of the restatement
(oracle/loss_oracle.py); check each decision branch on hand-built pixels; check that gh_image_loss rejects bad
arguments before launching anything, and its workspace size against the layout restated here."""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import loss64  # noqa: E402
import loss_oracle  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "loss64edges.npz")
PIN_TOL = 1e-12         # float64 against float64: a few units of 2^-53 of the scale
LAMBDAS = (0.8, 0.2, 0.4, 0.1)


def _worst(value, ref, scale):
    """max |value - ref| / scale; an element whose scale is 0 must match exactly."""
    value, ref, scale = (torch.as_tensor(np.asarray(a)).double() for a in (value, ref, scale))
    d = (value - ref).abs()
    assert bool((d[scale == 0] == 0).all()), "an element the replay calls exact differs"
    return float((d / scale.clamp(min=1e-300))[scale > 0].max())


@pytest.mark.parametrize("case", ["7x5", "1x13", "40x33"])
def test_replay_matches_reference_loss_utils_float64(case):
    with np.load(GOLDEN) as z:
        ins = [z[f"{case}/{k}"] for k in ("out", "gt_image", "gt_mask", "gt_angle", "gt_conf")]
        lam, want, dL = z["lambdas"], z[f"{case}/losses"], z[f"{case}/dL_dout"]
    r = loss64.replay(*ins, [float(x) for x in lam], consts=loss64.CONST64)
    assert not r["nan"]
    for k, v in zip(loss64.LOSSES, want):
        assert abs(r["losses"][k] - v) <= PIN_TOL * r["losses_scale"][k], k
    assert _worst(r["dL"], dL, r["scale"]) <= PIN_TOL
    # what the case exists to reach
    if case != "1x13":
        assert int((r["scale"][5:7] == 0).sum()) > 0 and float(r["dL"][6].abs().max()) > 1e6   # ties, eps gradient
    assert bool((r["scale"][[7, 9]] == 0).all())


@pytest.mark.parametrize("W,H,seed", [(45, 37, 1), (20, 18, 3), (33, 12, 5)])
def test_replay_matches_float64_autograd(W, H, seed):
    ins = loss_oracle.synthetic_case(W, H, seed)
    r = loss64.replay(*ins, LAMBDAS, consts=loss64.CONST64)
    x = ins[0].double().requires_grad_(True)
    loss, parts = loss_oracle.training_loss(x, *[t.double() for t in ins[1:]], *[float(np.float32(v)) for v in LAMBDAS])
    loss.backward()
    assert _worst(r["dL"], x.grad, r["scale"]) <= PIN_TOL
    assert abs(r["losses"]["total"] - float(loss.detach())) <= PIN_TOL * r["losses_scale"]["total"]
    for k in ("Ll1", "Lssim", "Lmask", "Lorient"):
        assert abs(r["losses"][k] - float(parts[k])) <= PIN_TOL * r["losses_scale"][k], k


def _one_pixel(c5, c6, conf=0.5, ang=0.3, m0=1.0, w=0.5):
    out = torch.zeros(10, 1, 1)
    out[5, 0, 0], out[6, 0, 0], out[8, 0, 0] = c5, c6, conf
    gm = torch.tensor([m0, 1.0]).reshape(2, 1, 1)
    return out, torch.zeros(3, 1, 1), gm, torch.full((1, 1, 1), ang), torch.full((1, 1, 1), w)


def test_replay_decisions_by_hand():
    """One pixel per branch of the orientation path, its gradient from the closed forms (lambda_orient = 1, so
    up = m0 w / sum(w) = 1)."""
    lam = (0.0, 0.0, 0.0, 1.0)
    # eps branch: zero direction, t = 0, ang = 0.5, mirror +1; d0 = 0.2 > 0, l0 = 0.2 < 0.8: dL/dc6 = -conf / eps
    r = loss64.replay(*_one_pixel(0.0, 0.0, conf=0.5, ang=0.3), lam)
    assert float(r["dL"][5]) == 0.0
    assert float(r["dL"][6]) == pytest.approx(-0.5 / loss64.EPS, rel=1e-15)
    assert float(r["ratios"]["eps"]) == math.inf and float(r["ratios"]["s0"]) > 1e6
    # nrm == eps exactly (c6 = 0): the nrm >= eps branch, c5^2 / nrm^3 = 1 / eps -- the same value
    r = loss64.replay(*_one_pixel(loss64.EPS, 0.0, conf=0.5, ang=0.3), lam)
    assert float(r["dL"][6]) == pytest.approx(-0.5 / loss64.EPS, rel=1e-12) and float(r["ratios"]["eps"]) == math.inf
    # clamp: c5 = 0.01, c6 = 1 clamps (nothing flows); c5 = 0.6, c6 = 0.8 passes, dL/dc6 = -conf * S * c5^2 / nrm^3 / sqrt(1 - t^2)
    r = loss64.replay(*_one_pixel(0.01, 1.0), lam)
    assert float(r["dL"][5]) == 0.0 and float(r["dL"][6]) == 0.0 and float(r["scale"][5]) == 0.0
    c5, c6 = float(np.float32(0.6)), float(np.float32(0.8))
    n = math.hypot(c5, c6)
    t = c6 / n
    ang = math.acos(t) / math.pi                                   # ~0.205; gt 0.3: d0 < 0, l0 is the minimum
    r = loss64.replay(*_one_pixel(c5, c6, conf=0.5, ang=0.3), lam)
    want6 = -0.5 * (-1.0) * c5 * c5 / n ** 3 / math.sqrt(1 - t * t)
    assert ang < float(np.float32(0.3)) and float(r["dL"][6]) == pytest.approx(want6, rel=1e-12)
    # mirror: c5 < 0 flips t and the sign of the derivative; c5 = -0.0 does not mirror
    r = loss64.replay(*_one_pixel(-c5, c6, conf=0.5, ang=0.9), lam)
    t2 = -t                                                         # ang = acos(-t) / pi ~0.795 < 0.9
    want6 = -0.5 * (-1.0) * (-1.0) * c5 * c5 / n ** 3 / math.sqrt(1 - t2 * t2)
    assert float(r["dL"][6]) == pytest.approx(want6, rel=1e-12)
    r0 = loss64.replay(*_one_pixel(-0.0, 0.0, conf=0.5, ang=0.3), lam)
    assert float(r0["dL"][6]) == pytest.approx(-0.5 / loss64.EPS, rel=1e-15)   # same as +0.0: not mirrored
    # torch.minimum ties: ang = 0.5 exactly; gt 0 -> l0 = l1 (0.5 each: +1 and -1 cancel), gt 0.5 -> d0 = 0, sign 0
    for gt in (0.0, 0.5, 1.0):
        r = loss64.replay(*_one_pixel(1.0, 0.0, conf=0.5, ang=gt), lam)
        assert float(r["dL"][5]) == 0.0 and float(r["dL"][6]) == 0.0 and float(r["scale"][6]) == 0.0, gt
        assert all(float(v) == math.inf for v in r["ratios"].values()), gt
    # a near tie gets an alternative: gt = 0.5 + 1e-7 puts d0 within float32 error of 0
    r = loss64.replay(*_one_pixel(c5, c6, conf=0.5, ang=ang + 1e-9), lam)
    assert float(r["ratios"]["s0"]) < loss64.DECISION_SAFETY and (0, 0) in r["alternatives"]
    names, vals = r["alternatives"][(0, 0)]
    assert "s0" in names and len({round(v[1], 6) for v in vals}) == 3        # sign -1, 0, +1
    # image / mask signs: I == G and mask == gt_mask give 0, sign(d) elsewhere
    out, gi, gm, ga, gc = _one_pixel(0.3, 0.4)
    out[0:3] = 0.5
    gi[0], gi[1], gi[2] = 0.5, 0.25, 0.75
    out[3], out[4] = gm[0], 0.25
    r = loss64.replay(out, gi, gm, ga, gc, (1.0, 0.0, 1.0, 0.0))
    assert [float(r["dL"][c]) for c in range(5)] == [0.0, 1.0 / 3.0, -1.0 / 3.0, 0.0, -0.5]


def test_replay_nan_guard_through_a_pixel():
    """gt_mask[0] = 0 with conf = -1e-7: log(conf + 1e-7) = log 0, times the zero mask, is NaN -> Lorient = 0 and no
    gradient flows into channels 5, 6, 8."""
    ins = list(loss64.edge_scene(9, 8, 4, specials=False))
    ins[0][8, 3, 4] = -float(np.float32(1e-7))
    ins[2][0, 3, 4] = 0.0
    r = loss64.replay(*ins, LAMBDAS)
    assert r["nan"] and r["losses"]["Lorient"] == 0.0
    assert bool((r["dL"][[5, 6, 8]] == 0).all()) and bool((r["scale"][[5, 6, 8]] == 0).all())
    assert float(r["dL"][0:5].abs().max()) > 0


def test_replay_crop_equals_full_replay():
    ins = loss64.edge_scene(61, 47, 6)
    full = loss64.replay(*ins, LAMBDAS)
    for x0, y0, x1, y1 in ((0, 0, 7, 9), (40, 30, 61, 47), (20, 11, 33, 25)):
        c = loss64.replay_crop(ins, LAMBDAS, x0, y0, x1, y1, full["sum_w"])
        ref = full["dL"][:, y0:y1, x0:x1]
        assert torch.allclose(c["dL"], ref, rtol=1e-13, atol=0) and torch.allclose(c["scale"], full["scale"][:, y0:y1, x0:x1], rtol=1e-12)
    s = loss64.chunked_sums(ins, LAMBDAS, rows=8)
    for k in loss64.SUMS:
        assert s["sums"][k] == pytest.approx(full["sums"][k], rel=1e-13, abs=1e-300)


# ------------------------------------------------------------------------------------------------ the C entry point
@pytest.fixture(scope="module")
def lib():
    from gaussianhaircut_b200 import build, _capi
    build.build(verbose=False)
    return _capi.load()


def _call(lib, W, H, ptrs, ws):
    out, gi, gm, ga, gc, losses, dL = ptrs
    return lib.gh_image_loss(W, H, out, gi, gm, ga, gc, 1.0, 1.0, 1.0, 1.0, ws, losses, dL, None, 0)


def test_image_loss_rejects_before_launching(lib):
    """Sizes, a missing pointer, a misaligned workspace and an image past 2^27 pixels are refused before any CUDA
    call.  Every call here fails one check, so no pointer is ever dereferenced."""
    from gaussianhaircut_b200 import _capi
    launches0 = lib.gh_kernel_launch_count()
    fake = C.c_void_p(0x10000)
    ptrs = [fake] * 7
    for W, H in ((0, 5), (5, 0), (-1, 5), (5, -3)):
        assert _call(lib, W, H, ptrs, fake) == _capi.GH_E_INVALID_ARG
        assert b"bad size" in lib.gh_last_error()
    for i in range(7):
        p = list(ptrs)
        p[i] = None
        assert _call(lib, 4, 4, p, fake) == _capi.GH_E_INVALID_ARG and b"missing pointer" in lib.gh_last_error()
    assert _call(lib, 4, 4, ptrs, None) == _capi.GH_E_INVALID_ARG
    assert _call(lib, 4, 4, ptrs, C.c_void_p(0x10004)) == _capi.GH_E_INVALID_ARG
    assert b"8-byte aligned" in lib.gh_last_error()
    # W * H = 2^27 + 1 = 81 * 19 * 87211, and a larger image
    assert 1539 * 87211 == (1 << 27) + 1
    assert _call(lib, 1539, 87211, ptrs, fake) == _capi.GH_E_INVALID_ARG
    assert b"2^27" in lib.gh_last_error()
    assert _call(lib, 1 << 16, 1 << 16, ptrs, fake) == _capi.GH_E_INVALID_ARG
    assert lib.gh_kernel_launch_count() == launches0


def _workspace_bytes(W, H):
    """gh_image_loss's workspace restated: 16 doubles of sums and tickets, one double per CTA of the presum (capped at
    132 * 8), three per CTA of the pointwise kernel (capped at 132 * 16) and one per 32x32 SSIM tile, then nine float
    maps of the image (three derivative maps per colour channel)."""
    n = W * H
    rb = min((n + 255) // 256, 1056)
    pb = min((n + 255) // 256, 2112)
    mb = ((W + 31) // 32) * ((H + 31) // 32)
    return (16 + rb + 3 * pb + mb) * 8 + 9 * n * 4


@pytest.mark.parametrize("W,H", [(1, 1), (1, 37), (37, 1), (255, 256), (256, 256), (257, 256), (270337, 1),
                                 (270336, 1), (77239, 7), (2112 * 256, 1), (1920, 1080), (16384, 8192)])
def test_image_loss_workspace_size(lib, W, H):
    n = C.c_size_t()
    assert lib.gh_image_loss_workspace_size(W, H, C.byref(n)) == 0
    assert n.value == _workspace_bytes(W, H)
    assert lib.gh_image_loss_workspace_size(0, H, C.byref(n)) != 0
