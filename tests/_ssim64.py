"""TEST INFRASTRUCTURE ONLY -- a float64 replay of the evaluation SSIM and PSNR (gh_eval_ssim) with first-order bounds
of a float32 evaluation in the kernel's operation order.

    ssim   loss_utils.ssim(img1, img2) with size_average (src/utils/loss_utils.py:72-121): the reference's own 11x11
           window (float32 1-D taps, float32 outer product; oracle/loss64.window) in float64, zero padding 5, the
           mean of ssim_map over 3 H W
    psnr   image_utils.psnr (src/utils/image_utils.py:17-19) on a (1,3,H,W) image: 20 log10(1 / sqrt(mse))

Inputs are the float32 values the kernel filters (after the uint8 conversion and the clamps); `mask` (1,H,W) is
multiplied into both images, one float32 rounding each.

Bounds (units of u = 2^-24, the running error analysis of oracle/loss64.V).  A window sum is formed separably: 11
FMAs along the row, then 11 along the column, each rounding once to at most u times the sum of the absolute terms,
and the separable taps g_i g_j differ from the reference's float32 outer product by at most u each, so

    e(conv(x)) = conv(e(x)) + 23 conv(|x|)

The per-pixel map is gh_image_math.cuh's gh_ssim_pixel<true>: mu^2 and mu1 mu2, sigma = E - mu^2, a1 = 2 mu12 + C1,
a2 = 2 sigma12 + C2, b1 = mu1^2 + mu2^2 + C1, b2 = sigma1 + sigma2 + C2, S = (a1 a2) / (b1 b2), every operation
rounded once; C1 = fl(fl(0.01)^2), C2 = fl(fl(0.03)^2) sit within 3 u of
0.01^2, 0.03^2.  The sum over the pixels is in double (N 2^-53 relative) and the mean is rounded to float32 once.
PSNR: d = fl(x - y) (one rounding), d^2 and the sum in double, so mse is within 2 u relative (+ the double sum);
psnr = -10 log10(mse) moves by 10 / ln 10 times that, and is rounded to float32 once.
"""
from __future__ import annotations

import math
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
from loss64 import V, conv, window  # noqa: E402

U = 2.0 ** -24
C1, C2 = 0.01 ** 2, 0.03 ** 2
CONV_ROUNDINGS = 23
CONST_E = 3.0                          # bound of the float32 constants C1, C2 (units of u, relative)


def _f64(a, device):
    if isinstance(a, np.ndarray):
        a = torch.from_numpy(np.ascontiguousarray(a))
    return a.to(device=device, dtype=torch.float64)


def _conv(a: V, w) -> V:
    return V(conv(a.v, w), conv(a.e, w) + CONV_ROUNDINGS * conv(a.v.abs(), w))


def _const(c, like, e=CONST_E):
    return V(torch.full_like(like, c), torch.full_like(like, e * c))


def replay(img1, img2, mask=None, device=None) -> dict:
    """img1, img2 (3,H,W), mask (1,H,W) or None: float32 values as arrays or tensors.  -> {ssim, ssim_scale, psnr,
    psnr_scale, mse, ssim_map}: the float64 values, and the bounds in units of u (|float32 - replay| <= u * scale)."""
    if device is None:
        device = img1.device if isinstance(img1, torch.Tensor) else torch.device("cpu")
    x, y = V(_f64(img1, device)), V(_f64(img2, device))
    if mask is not None:
        m = V(_f64(mask, device).expand_as(x.v))
        x, y = x * m, y * m
    w = window(device)
    n = x.v.numel()
    mu1, mu2 = _conv(x, w), _conv(y, w)
    e11, e22, e12 = _conv(x * x, w), _conv(y * y, w), _conv(x * y, w)
    mu1_sq, mu2_sq, mu12 = mu1 * mu1, mu2 * mu2, mu1 * mu2
    s1, s2, s12 = e11 - mu1_sq, e22 - mu2_sq, e12 - mu12
    a1, a2 = 2.0 * mu12 + _const(C1, x.v), 2.0 * s12 + _const(C2, x.v)
    b1, b2 = mu1_sq + mu2_sq + _const(C1, x.v), s1 + s2 + _const(C2, x.v)
    S = (a1 * a2) / (b1 * b2)
    ssim = float(S.v.sum()) / n
    double_sum = n * 2.0 ** -53 / U                 # the double sum, relative to the sum of |S|, in units of u
    ssim_scale = float(S.e.sum()) / n + abs(ssim) + double_sum * float(S.v.abs().sum()) / n
    d = x.v - y.v
    mse = float((d * d).sum()) / n
    with np.errstate(divide="ignore"):
        psnr = float(20.0 * np.log10(1.0 / np.sqrt(np.float64(mse))))
    psnr_scale = (10.0 / math.log(10.0)) * (2.0 + double_sum) + (abs(psnr) if math.isfinite(psnr) else 0.0)
    return dict(ssim=ssim, ssim_scale=ssim_scale, psnr=psnr, psnr_scale=psnr_scale, mse=mse, ssim_map=S.v)


def cases():
    """{name: (img1 (3,H,W), img2 (3,H,W), mask (1,H,W) or None)} float32: shapes smaller than the window, around it
    and beyond, constant images (sigma = 0), identical images, a render-like image with a large background, a masked
    pair, and values outside [0, 1]."""
    g = np.random.default_rng(22)
    r = lambda *s: g.uniform(0, 1, s).astype(np.float32)  # noqa: E731
    out = {}
    for H, W in ((1, 1), (5, 7), (10, 10), (11, 11), (17, 33), (64, 48)):
        a = r(3, H, W)
        out[f"rand_{H}x{W}"] = (a, np.clip(a + g.normal(0, 0.1, a.shape).astype(np.float32), 0, 1), None)
    out["const"] = (np.full((3, 19, 23), 0.25, np.float32), np.full((3, 19, 23), 0.75, np.float32), None)
    out["const_equal"] = (np.full((3, 12, 9), 0.5, np.float32), np.full((3, 12, 9), 0.5, np.float32), None)
    a = r(3, 40, 37)
    out["identical"] = (a, a.copy(), None)
    # a render: a textured blob on a flat background (the background is most of the frame)
    H, W = 72, 96
    yy, xx = np.mgrid[0:H, 0:W]
    blob = (((yy - 30) / 14.0) ** 2 + ((xx - 50) / 20.0) ** 2 < 1).astype(np.float32)
    bg = np.array([0.1, 0.2, 0.3], np.float32)[:, None, None]
    tex = r(3, H, W)
    ren = (blob * tex + (1 - blob) * bg).astype(np.float32)
    gt = (blob * np.clip(tex + g.normal(0, 0.05, tex.shape), 0, 1) + (1 - blob) * bg).astype(np.float32)
    out["render_bg"] = (ren, gt, None)
    out["masked"] = (r(3, 33, 29), r(3, 33, 29), (r(1, 33, 29) > 0.4).astype(np.float32) * r(1, 33, 29))
    out["outside01"] = (g.uniform(-0.2, 1.2, (3, 21, 18)).astype(np.float32), r(3, 21, 18), None)
    return out
