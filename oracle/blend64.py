"""TEST INFRASTRUCTURE ONLY -- a float64 replay of the tile blend, forward and backward.

The product never imports this.  Given the per-Gaussian 2-D state (means2D, conic/opacity), the colours, the
background, the per-tile sorted lists (point_list + ranges) and dL/dpix, `replay` recomputes what the reference's
renderCUDA kernels compute (forward.cu:356-394, backward.cu:490-558), every pixel taking the reference's decisions in
list order:

    skip when power > 0;  skip when alpha < 1/255;  alpha capped at 0.99;  stop when test_T = T (1 - alpha) < 1e-4

Decisions and magnitudes are evaluated in float64 from the float32 inputs, against the float32 constants the kernels
compare with (1.0f / 255.0f, 0.99f, 0.0001f), so the replay is the exact-arithmetic value of the reference's formula.
A float32 kernel can only take a different decision where the exact value lies within float32's error of the
threshold.  The replay therefore also returns every reached decision's margin to its threshold, divided by the
first-order float32 error bound derived below; a scene on which every such ratio is comfortably above 1 has exactly
one correct set of decisions, and the kernels' n_contrib must equal the replay's bit for bit.

Float32 error bounds (u = 2^-24, first order; the tests ask for a ratio of at least DECISION_SAFETY):

  power = fma(fma(dx, dx*a, dy*(dy*c)), -0.5, -(dy*(dx*b))),  dx = fl(x - px), dy = fl(y - py)   (gh_power)
      a dx^2 carries 3 roundings (dx twice, dx*a), c dy^2 four, b dx dy four, the inner fma one on |a dx^2| + |c dy^2|
      and the outer fma one on |power|.  With M = |a dx^2| / 2 + |c dy^2| / 2 + |b dx dy|:
          |d power| <= 6 u M.
  G = expf(power): CUDA's expf is within 2 ulp (<= 4 u relative), plus the propagated |d power|.
  alpha = min(0.99f, op * G): one more rounding.        |d alpha| / alpha <= eps_a = (6 M + 5) u.
      The cap is exact: alpha = 0.99f in both wherever op G exceeds 0.99f by more than eps_a.
  1 - alpha: exact for alpha >= 1/2 (Sterbenz), else one rounding; alpha's own error enters amplified by
      alpha / (1 - alpha) unless alpha is capped.  Each product T (1 - alpha) rounds once more.  Over the records a
      pixel has multiplied in up to record k:
          |d T_k| / T_k <= eps_T,k = sum_i (eps_a,i alpha_i / (1 - alpha_i) [uncapped] + 2 u).
      (The reference's own figure: T drifts by about n * 1.2e-7 over n records.)

  alpha decision   (power <= 0):              ratio = |alpha / (1/255)f - 1| / eps_a
  power decision   (M > 0; M == 0 is exact):  ratio = |power| / (6 u M)
  stop decision    (alpha passed):            ratio = |test_T / 1e-4f - 1| / eps_T,k

Only decisions a pixel actually reaches count: every record up to and including the one it stops on.

Gradients are returned in the reference binding's layouts (rasterize_points.cu:160-168): dL_dmeans2D (P,3) with the
W/2 and H/2 factors and a zero z, dL_dcolors (P,C), dL_dopacity (P,1), dL_dconic (P,2,2) with [1,0] zero.  For every
Gaussian and component the replay also returns a scale: the sum over its (pixel, Gaussian) terms of the term's
magnitude with every sum inside it taken in absolute value (dL/dalpha's colour, suffix and background parts
included).  A float32 implementation's error in a component is a small multiple of that scale, whatever cancels.
"""
from __future__ import annotations

import numpy as np
import torch

U = 2.0 ** -24
ALPHA_MIN = float(np.float32(1.0 / 255.0))
ALPHA_MAX = float(np.float32(0.99))
T_MIN = float(np.float32(0.0001))
DECISION_SAFETY = 4.0      # the tests' least margin / bound ratio: covers the O(u^2) terms the bounds leave out
BLOCK = 16


def _t(a, device, dtype=torch.float64):
    if isinstance(a, np.ndarray):
        a = torch.from_numpy(np.ascontiguousarray(a))
    return a.to(device=device, dtype=dtype)


def replay(means2D, conic_opacity, colors, bg, point_list, ranges, W: int, H: int, dL_dpix=None, device=None) -> dict:
    """means2D (P,2), conic_opacity (P,4) = (a, b, c, opacity), colors (P,C), bg (C,), point_list (R,) Gaussian index
    per record, ranges (T,2) per-tile [start, end) in row-major tile order, dL_dpix (C,H,W) or None (forward only).
    numpy arrays or tensors; the replay runs in float64 on `device` (default: that of means2D when it is a tensor).

    Returns image (C,H,W), final_T (H*W), n_contrib (H*W) int64, stopped (H*W, the pixel took the test_T stop),
    and when dL_dpix is given dL_dmeans2D, dL_dcolors,
    dL_dopacity, dL_dconic plus `scale` (same keys and shapes) and `image_scale` (C,H,W).  Decision margins:
    alpha_ratio / power_ratio / stop_ratio (least margin / bound over every reached decision, inf if none) and
    alpha_rel (float64, every reached alpha decision's alpha / (1/255)f - 1, for scenes that count near-threshold
    pairs)."""
    if device is None:
        device = means2D.device if isinstance(means2D, torch.Tensor) else torch.device("cpu")
    f64 = lambda a: _t(a, device)   # noqa: E731
    xy, co, col, bgv = f64(means2D), f64(conic_opacity), f64(colors), f64(bg)
    pl = _t(point_list, device, torch.int64)
    rg = _t(ranges, device, torch.int64).reshape(-1, 2)
    P, C = col.shape[0], col.shape[1]
    gx = (W + BLOCK - 1) // BLOCK
    image = bgv[:, None].repeat(1, H * W)              # an empty tile shows the background (T = 1)
    final_T = torch.ones(H * W, dtype=torch.float64, device=device)
    n_contrib = torch.zeros(H * W, dtype=torch.int64, device=device)
    stopped = torch.zeros(H * W, dtype=torch.bool, device=device)
    backward = dL_dpix is not None
    if backward:
        dpix = f64(dL_dpix).reshape(C, H * W)
        acc = torch.zeros(P, 16, dtype=torch.float64, device=device)      # colours, mean2D x y, conic x y w, opacity
        acc_s = torch.zeros(P, 16, dtype=torch.float64, device=device)
        image_scale = bgv.abs()[:, None].repeat(1, H * W)
    ratios = {"alpha_ratio": [], "power_ratio": [], "stop_ratio": []}
    alpha_rel = []
    by, bx = torch.meshgrid(torch.arange(BLOCK, device=device), torch.arange(BLOCK, device=device), indexing="ij")
    lens = (rg[:, 1] - rg[:, 0]).cpu().numpy()
    for tile in np.nonzero(lens)[0].tolist():
        r0, r1 = int(rg[tile, 0]), int(rg[tile, 1])
        ty, tx = divmod(tile, gx)
        px, py = (tx * BLOCK + bx).reshape(-1), (ty * BLOCK + by).reshape(-1)
        inside = (px < W) & (py < H)
        px, py = px[inside].double(), py[inside].double()
        pix = (py * W + px).long()
        ids = pl[r0:r1]
        g = xy[ids]
        a, b, c, op = co[ids, 0], co[ids, 1], co[ids, 2], co[ids, 3]
        # (pixels x records)
        dx = g[None, :, 0] - px[:, None]
        dy = g[None, :, 1] - py[:, None]
        q1, q2, q3 = a * dx * dx, c * dy * dy, b * dx * dy
        power = -0.5 * (q1 + q2) - q3
        M = 0.5 * q1.abs() + 0.5 * q2.abs() + q3.abs()
        G = torch.exp(power)
        x = op * G
        alpha = torch.clamp(x, max=ALPHA_MAX)
        ok = ~(power > 0) & ~(alpha < ALPHA_MIN)
        eps_a = (6.0 * M + 5.0) * U
        # stop: the first record that passes and takes T below 1e-4 (T only falls, so a cumulative product of every
        # passing record is exact up to and including it)
        om = torch.where(ok, 1.0 - alpha, torch.ones_like(alpha))
        T_incl = torch.cumprod(om, dim=1)
        stops = ok & (T_incl < T_MIN)
        L = ids.shape[0]
        idx = torch.arange(L, device=device)
        stop_at = torch.where(stops.any(dim=1), torch.where(stops, idx, L).min(dim=1).values, torch.full_like(pix, L))
        reached = idx[None, :] <= stop_at[:, None]
        blended = ok & (idx[None, :] < stop_at[:, None])
        # decision margins
        dec = reached & ~(power > 0)
        alpha_rel.append((alpha / ALPHA_MIN - 1.0)[dec])
        ratios["alpha_ratio"].append(((alpha / ALPHA_MIN - 1.0).abs() / eps_a)[dec])
        pw = reached & (M > 0)
        ratios["power_ratio"].append((power.abs() / (6.0 * U * M))[pw])
        uncapped = x < ALPHA_MAX * (1.0 + eps_a)
        drift = torch.where(ok, eps_a * alpha / (1.0 - alpha) * uncapped + 2.0 * U, torch.zeros_like(alpha))
        eps_T = torch.cumsum(drift, dim=1)
        st = ok & reached
        ratios["stop_ratio"].append(((T_incl / T_MIN - 1.0).abs() / eps_T)[st])
        # forward
        ab = torch.where(blended, alpha, torch.zeros_like(alpha))
        T_after = torch.cumprod(1.0 - ab, dim=1)
        T_before = torch.cat([torch.ones_like(T_after[:, :1]), T_after[:, :-1]], dim=1)
        w = ab * T_before                                   # d(pixel) / d(colour)
        Tf = T_after[:, -1]
        feat = col[ids]
        image[:, pix] = (w @ feat).T + Tf[None, :] * bgv[:, None]
        final_T[pix] = Tf
        n_contrib[pix] = torch.where(blended, idx + 1, 0).max(dim=1).values
        stopped[pix] = stop_at < L
        if not backward:
            continue
        image_scale[:, pix] = (w @ feat.abs()).T + Tf[None, :] * bgv.abs()[:, None]
        d = dpix[:, pix].T                                  # (pixels x C)
        cd, cd_abs = d @ feat.T, d.abs() @ feat.abs().T     # c . dL per (pixel, record)
        bgd, bgd_abs = d @ bgv, d.abs() @ bgv.abs()
        # suffix of the colour blended behind each record, over T after it (backward.cu:519-523):
        #   sum_ch accum_rec[ch] dL[ch] = sum_{j > k} w_j (c_j . dL) / T_after_k
        def behind(v):
            s = torch.flip(torch.cumsum(torch.flip(w * v, [1]), dim=1), [1])
            return torch.cat([s[:, 1:], torch.zeros_like(s[:, :1])], dim=1) / torch.where(blended, T_after, torch.ones_like(T_after))
        dL_dalpha = T_before * (cd - behind(cd)) - Tf[:, None] / (1.0 - ab) * bgd[:, None]
        mag = T_before * (cd_abs + behind(cd_abs)) + Tf[:, None] / (1.0 - ab) * bgd_abs[:, None]
        Gb = torch.where(blended, G, torch.zeros_like(G))
        dL_dG, mag_G = op * dL_dalpha, op.abs() * mag
        gdx, gdy = Gb * dx, Gb * dy
        terms = [
            (dL_dG * (-gdx * a - gdy * b) * (0.5 * W), mag_G * (gdx * a).abs() + mag_G * (gdy * b).abs()),
            (dL_dG * (-gdy * c - gdx * b) * (0.5 * H), mag_G * (gdy * c).abs() + mag_G * (gdx * b).abs()),
            (-0.5 * gdx * dx * dL_dG, 0.5 * (gdx * dx).abs() * mag_G),
            (-0.5 * gdx * dy * dL_dG, 0.5 * (gdx * dy).abs() * mag_G),
            (-0.5 * gdy * dy * dL_dG, 0.5 * (gdy * dy).abs() * mag_G),
            (Gb * dL_dalpha, Gb * mag),
        ]
        acc[ids, :C] += w.T @ d
        acc_s[ids, :C] += w.T @ d.abs()
        for k, (t, s) in enumerate(terms):
            acc[ids, C + k] += t.sum(dim=0)
            acc_s[ids, C + k] += (s * (0.5 * W if k == 0 else 0.5 * H if k == 1 else 1.0)).sum(dim=0)
    out = {"image": image.reshape(C, H, W), "final_T": final_T, "n_contrib": n_contrib, "stopped": stopped}
    for k, v in ratios.items():
        v = torch.cat(v) if v else torch.zeros(0, dtype=torch.float64, device=device)
        out[k] = float(v.min()) if v.numel() else float("inf")
    out["alpha_rel"] = torch.cat(alpha_rel) if alpha_rel else torch.zeros(0, dtype=torch.float64, device=device)
    if backward:
        out.update(_layout(acc, C))
        out["scale"] = _layout(acc_s, C)
        out["image_scale"] = image_scale.reshape(C, H, W)
    return out


def _layout(a: torch.Tensor, C: int) -> dict:
    """[P][C + 6] accumulators -> the reference binding's gradient layouts."""
    P = a.shape[0]
    z = torch.zeros(P, dtype=a.dtype, device=a.device)
    return {"dL_dcolors": a[:, :C].clone(),
            "dL_dmeans2D": torch.stack([a[:, C], a[:, C + 1], z], dim=1),
            "dL_dconic": torch.stack([a[:, C + 2], a[:, C + 3], z, a[:, C + 4]], dim=1).reshape(P, 2, 2),
            "dL_dopacity": a[:, C + 5:C + 6].clone()}


GRADS = ("dL_dmeans2D", "dL_dcolors", "dL_dopacity", "dL_dconic")


def worst_ratio(value, ref: torch.Tensor, scale: torch.Tensor, floor: float) -> float:
    """max over elements of |value - ref| / (scale + floor): the least tol with |value - ref| <= tol (scale + floor)
    everywhere."""
    v = _t(value, ref.device).reshape(ref.shape)
    return float(((v - ref).abs() / (scale + floor)).max()) if ref.numel() else 0.0
