"""TEST INFRASTRUCTURE ONLY -- a float64 replay of the appearance-stage loss and its gradient w.r.t. the render.

The product never imports this.  Given the float32 render (10,H,W), the supervision maps and the four lambdas,
`replay` evaluates the reference's training loss (SRC/train_gaussians.py:126-140 with SRC/utils/loss_utils.py and the
dir -> angle step of SRC/gaussian_renderer/__init__.py:98-105) in float64 and differentiates it by hand:

  * the 11x11 window is the reference's own 2-D window (create_window: float32 1-D taps, float32 normalisation, float32
    outer product), widened to float64; every convolution is zero-padded and written as 121 shifted adds, so no cuDNN
    algorithm or TF32 setting enters the replay;
  * F.normalize: den = max(nrm, eps) with eps = float32(1e-12); its backward takes the constant-denominator branch only
    where nrm < eps (clamp_min passes the gradient where nrm >= eps);
  * mirror where dir.x < 0 (so c5 = -0.0 is not mirrored); clamp to [-1 + 1e-3, 1 - 1e-3], passing the gradient where
    the input lies inside, bounds included; torch.minimum splits the gradient evenly on a tie; sign(0) = 0;
  * conf + 1e-7 with the float32 constant (a conf of exactly -1e-7 gives log 0); Lorient -> 0 when it is NaN, which
    zeroes channels 5, 6 and 8 of the gradient.

Scales.  Every value v of the replay carries e(v), a first-order bound of a float32 evaluation's error in units of
u = 2^-24, formed by running error analysis over the reference's operations:

    a +- b:  e = e_a + e_b + |a| + |b|          a * b:  e = |a| e_b + |b| e_a + |a b|
    a / b:   e = e_a / |b| + |a| e_b / b^2 + |a / b|       sqrt a:  e = e_a / (2 sqrt a) + |sqrt a|
    conv(x): e = conv(e_x) + conv(|x|)          (one rounding per window sum, whatever its order)

so every inner sum enters in absolute value, and a quotient divides its numerator's and denominator's bounds by the
denominator: this is where cancellation shows.  sigma = E[x^2] - mu^2, b2 = sigma1 + sigma2 + C2 and a2 = 2 sigma12 + C2
carry bounds of the size of E[x^2] + mu^2 while b2 itself can be as small as C2 = 9e-4; the map, its three derivative
maps and the image gradient inherit e(b2) / b2.  The replay returns these e as `scale`: a float32 implementation of the
same operation lies within a small multiple of u * scale of the replay, wherever it cancels.  The remaining terms:

  * acos: CUDA documents acosf within 2 ulp (<= 4 u relative); with the division by pi (a float32 constant, one more
    rounding, and the quotient's own) e(ang) = |acos'(t)| e(t) / pi + 6 |ang|.  acos(0) / pi is exactly 0.5 in float32
    (acosf(0) = fl(pi / 2) = fl(pi) / 2), so t == 0 with e(t) == 0 gives e(ang) = 0;
  * nrm = sqrt(c5^2 + c6^2): e = 2 nrm (two roundings under the root, halved, plus the root's); exact when c5 or c6 is
    zero (sqrt(fl(c^2)) = |c| in round-to-nearest while c^2 is a normal number);
  * 1 / sum(w): the orientation gradient and Lorient divide by the sum of gt_orient_conf; a float32 tree sum of N terms
    is within (1 + log2 N) u sum|w|, and that relative error enters every orientation gradient;
  * a loss sum over N pixels: e = sum e_i + (1 + log2 N) sum |t_i|.
  * An operation whose operands are exact and whose exact result is a float32 number is exact (e = 0).

Decisions.  mirror and the signs of I - G and of mask - gt_mask are exact (the float32 difference of two float32
numbers has the exact difference's sign).  The others are returned per pixel as margin / (u * bound):

    eps      |nrm - eps| / e(nrm)             clamp    min(|diry - lo|, |diry - hi|) / e(diry)
    outer    |l0 - min(l1, l2)| / (e(d0) + e(inner))   inner    |l1 - l2| / (e(d1) + e(d2))
    s0 s1 s2 |d_k| / e(d_k)

inf where the decision is exact (zero bound) or cannot change any output at that pixel.  Where a ratio is below
DECISION_SAFETY, `alternatives` lists every gradient (channels 5, 6) the pixel can have when the ambiguous decisions
go either way, so that a test can accept any of them and count such pixels.

Crops.  A pixel's gradient depends only on the inputs within 10 pixels (two 11-tap windows) and on sum(w): `replay_crop`
returns the gradient of a rectangle from the rectangle plus a 10-pixel halo, given the global sum of weights and the
image size, and `chunked_sums` forms the five sums of an image too large for one replay, in row bands.
"""
from __future__ import annotations

import itertools
import math

import numpy as np
import torch

U = 2.0 ** -24
DECISION_SAFETY = 4.0
HALO = 10
R = 5                                   # window radius
_f32 = lambda x: float(np.float32(x))   # noqa: E731
# the constants as a float32 evaluation sees them; CONST64: as a float64 evaluation of the reference sees them
CONST32 = {"eps": _f32(1e-12), "lo": _f32(-1 + 1e-3), "hi": _f32(1 - 1e-3), "e7": _f32(1e-7)}
CONST64 = {"eps": 1e-12, "lo": -1 + 1e-3, "hi": 1 - 1e-3, "e7": 1e-7}
EPS, LO, HI, E7 = (CONST32[k] for k in ("eps", "lo", "hi", "e7"))
C1, C2 = 0.01 ** 2, 0.03 ** 2
DECISIONS = ("eps", "clamp", "outer", "inner", "s0", "s1", "s2")
SUMS = ("w", "l1", "ssim", "mask", "orient")
LOSSES = ("total", "Ll1", "Lssim", "Lmask", "Lorient")


def window(device="cpu") -> torch.Tensor:
    """The reference's 11x11 window (loss_utils.py:81-89): float32 1-D taps, float32 normalisation, float32 outer
    product, returned in float64."""
    g = torch.Tensor([math.exp(-(x - 5) ** 2 / float(2 * 1.5 ** 2)) for x in range(11)])
    g = (g / g.sum()).unsqueeze(1)
    return g.mm(g.t()).float().double().to(device)


def conv(x: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    """Zero-padded 11x11 window sum over the last two dims, as 121 shifted adds (the window is symmetric, so this is
    also its adjoint)."""
    H, W = x.shape[-2:]
    xp = torch.nn.functional.pad(x, (R, R, R, R))
    out = torch.zeros_like(x)
    for i in range(11):
        for j in range(11):
            out += w[i, j] * xp[..., i:i + H, j:j + W]
    return out


def _exact32(x):
    return x == x.float().double()


class V:
    """A float64 value and its float32 error bound e (units of u); see the module docstring."""
    __slots__ = ("v", "e")

    def __init__(self, v, e=None):
        self.v = v
        self.e = torch.zeros_like(v) if e is None else e

    @staticmethod
    def c(x, like):
        return x if isinstance(x, V) else V(torch.full_like(like, float(x)), torch.full_like(like, abs(float(x))) * (
            0.0 if float(np.float32(x)) == float(x) else 1.0))

    def __add__(a, b):
        b = V.c(b, a.v)
        return V(a.v + b.v, a.e + b.e + a.v.abs() + b.v.abs())

    __radd__ = __add__

    def __sub__(a, b):
        b = V.c(b, a.v)
        return V(a.v - b.v, a.e + b.e + a.v.abs() + b.v.abs())

    def __rsub__(a, b):
        return V.c(b, a.v) - a

    def __mul__(a, b):
        b = V.c(b, a.v)
        v = a.v * b.v
        return V(v, a.v.abs() * b.e + b.v.abs() * a.e + v.abs())

    __rmul__ = __mul__

    def __truediv__(a, b):
        b = V.c(b, a.v)
        v = a.v / b.v
        return V(v, a.e / b.v.abs() + a.v.abs() * b.e / (b.v * b.v) + v.abs())

    def __neg__(a):
        return V(-a.v, a.e)

    def conv(a, w):
        return V(conv(a.v, w), conv(a.e, w) + conv(a.v.abs(), w))


def _sum(t: V, n: int) -> tuple:
    """A loss sum over n pixels and its bound."""
    return float(t.v.sum()), float(t.e.sum() + (1.0 + math.log2(max(n, 1))) * t.v.abs().sum())


def _ratio(margin, bound):
    r = margin / (U * bound)
    return torch.where(bound == 0, torch.full_like(r, math.inf), r)


# ------------------------------------------------------------------------------------------------ orientation
def _orient_base(c5, c6, conf, g, up, e_up, k):
    """Per-pixel quantities of the orientation path that do not depend on a decision (flat float64 tensors)."""
    EPS, LO, HI = k["eps"], k["lo"], k["hi"]
    nrm = torch.sqrt(c5 * c5 + c6 * c6)
    normal = nrm >= EPS
    one_zero = ((c5 == 0) & (c6.abs() >= 2.0 ** -60)) | ((c6 == 0) & (c5.abs() >= 2.0 ** -60)) | ((c5 == 0) & (c6 == 0))
    e_nrm = torch.where(one_zero, torch.zeros_like(nrm), 2.0 * nrm)
    den = torch.clamp(nrm, min=EPS)
    e_den = torch.where(normal, e_nrm, torch.zeros_like(nrm))
    diry = c6 / den
    exact_in = e_den == 0
    e_diry = c6.abs() * e_den / (den * den) + torch.where(exact_in & _exact32(diry), torch.zeros_like(diry), diry.abs())
    mirror = torch.where((c5 / den).float() < 0, -1.0, 1.0).double()
    passes = (diry >= LO) & (diry <= HI)
    t = torch.clamp(diry, LO, HI) * mirror
    e_t = torch.where(passes, e_diry, torch.zeros_like(e_diry))
    acos = torch.acos(t)
    ang = acos / math.pi
    dacos = 1.0 / torch.sqrt(1.0 - t * t)
    e_ang = torch.where((t == 0) & (e_t == 0), torch.zeros_like(t), dacos * e_t / math.pi + 6.0 * ang.abs())
    d0 = ang - g
    e_d0 = e_ang + torch.where((e_ang == 0) & _exact32(d0), torch.zeros_like(d0), d0.abs())
    d1, d2 = d0 - 1.0, d0 + 1.0
    e_d1 = e_d0 + torch.where((e_d0 == 0) & _exact32(d1), torch.zeros_like(d1), d1.abs())
    e_d2 = e_d0 + torch.where((e_d0 == 0) & _exact32(d2), torch.zeros_like(d2), d2.abs())
    l0, l1, l2 = d0.abs(), d1.abs(), d2.abs()
    # sqrt(1 - t^2): bound of 1 - t^2, then the root
    q = 1.0 - t * t
    e_q = 2.0 * t.abs() * e_t + t * t + 1.0 + t * t
    sq = torch.sqrt(q)
    e_sq = e_q / (2.0 * sq) + sq
    return dict(eps=EPS, c5=c5, c6=c6, conf=conf, up=up, e_up=e_up, nrm=nrm, e_nrm=e_nrm, normal=normal, diry=diry,
                e_diry=e_diry, mirror=mirror, passes=passes, t=t, e_t=e_t, d0=d0, d1=d1, d2=d2, e_d0=e_d0, e_d1=e_d1,
                e_d2=e_d2, l0=l0, l1=l1, l2=l2, sq=sq, e_sq=e_sq)


def _tri(a, b):
    """torch.minimum(a, b)'s gradient weight on a: 1, 0.5 on a tie, 0."""
    return torch.where(a < b, 1.0, torch.where(a == b, 0.5, 0.0)).double()


def _decide(b):
    """The reference's decisions on the exact values."""
    inner = torch.minimum(b["l1"], b["l2"])
    return dict(eps=~b["normal"], clamp=b["passes"], outer=_tri(b["l0"], inner), inner=_tri(b["l1"], b["l2"]),
                s0=torch.sign(b["d0"]), s1=torch.sign(b["d1"]), s2=torch.sign(b["d2"]))


OPTIONS = {"eps": (False, True), "clamp": (False, True), "outer": (0.0, 0.5, 1.0), "inner": (0.0, 0.5, 1.0),
           "s0": (-1.0, 0.0, 1.0), "s1": (-1.0, 0.0, 1.0), "s2": (-1.0, 0.0, 1.0)}


def _orient_grad(b, d):
    """dL/dc5, dL/dc6 and their bounds for decisions d."""
    wo, w1 = d["outer"], d["inner"]
    S = wo * d["s0"] + (1.0 - wo) * (w1 * d["s1"] + (1.0 - w1) * d["s2"])
    pas = d["clamp"].double() if d["clamp"].dtype == torch.bool else d["clamp"]
    nrm, c5, c6 = b["nrm"], b["c5"], b["c6"]
    eps_b = d["eps"]
    safe = torch.where(eps_b, torch.ones_like(nrm), nrm)
    inv3 = 1.0 / (safe * safe * safe)
    ddy5 = torch.where(eps_b, torch.zeros_like(nrm), -c5 * c6 * inv3)
    ddy6 = torch.where(eps_b, torch.full_like(nrm, 1.0 / b["eps"]), c5 * c5 * inv3)
    rel_ddy = torch.where(eps_b, torch.ones_like(nrm), 3.0 * (b["e_nrm"] / safe + 1.0) + 2.0)
    common = -b["up"] * b["conf"] * S * b["mirror"] * pas / b["sq"]
    # relative bound of the common factor: up, conf * pi, the signs' sum (exact), 1 / (pi sqrt(1 - t^2)), products
    rel = b["e_up"] / b["up"].abs().clamp(min=1e-300) + 2.0 + b["e_sq"] / b["sq"] + 2.0 + 4.0
    g5, g6 = common * ddy5, common * ddy6
    return g5, g6, g5.abs() * (rel + rel_ddy), g6.abs() * (rel + rel_ddy)


def _orient(c5, c6, conf, g, m0, w, lam, sum_w, e_sum_w, k):
    """Per-pixel orientation: the loss term, dL/d(c5, c6, conf) with bounds, decision ratios, alternatives."""
    EPS, LO, HI, E7 = k["eps"], k["lo"], k["hi"], k["e7"]
    inv = 1.0 / sum_w if sum_w != 0 else math.inf
    rel_sw = e_sum_w / abs(sum_w) if sum_w != 0 else math.inf
    with np.errstate(all="ignore"):
        up = m0 * w * (lam * inv)
    e_up = up.abs() * (rel_sw + 4.0)
    b = _orient_base(c5, c6, conf, g, up, e_up, k)
    d = _decide(b)
    g5, g6, e5, e6 = _orient_grad(b, d)
    # Lmin = pi min(l0, l1, l2); its bound follows the branch taken
    inner = torch.minimum(b["l1"], b["l2"])
    e_inner = torch.where(b["l1"] < b["l2"], b["e_d1"], torch.where(b["l1"] > b["l2"], b["e_d2"],
                                                                     torch.maximum(b["e_d1"], b["e_d2"])))
    lmin = torch.minimum(b["l0"], inner)
    e_lmin_raw = torch.where(b["l0"] < inner, b["e_d0"], torch.where(b["l0"] > inner, e_inner,
                                                                     torch.maximum(b["e_d0"], e_inner)))
    Lmin = V(lmin * math.pi, math.pi * e_lmin_raw + 2.0 * lmin * math.pi)
    q = V(conf + E7, torch.where(_exact32(conf + E7), 0.0, (conf + E7).abs()).double())
    with np.errstate(all="ignore"):
        logq = torch.log(q.v)
        Llog = V(logq, q.e / q.v.abs() + 2.0 * logq.abs())
        lp = (Lmin * V(conf) - Llog) * V(m0) * V(w)
        rq = V(1.0 / q.v, q.e / (q.v * q.v) + (1.0 / q.v).abs())
        g8 = V(up, e_up) * (Lmin - rq)
    # decision ratios, inf where the decision cannot change an output
    ratios = {
        "eps": _ratio((b["nrm"] - EPS).abs(), b["e_nrm"]),
        "clamp": _ratio(torch.minimum((b["diry"] - LO).abs(), (b["diry"] - HI).abs()), b["e_diry"]),
        "outer": _ratio((b["l0"] - inner).abs(), b["e_d0"] + e_inner),
        "inner": _ratio((b["l1"] - b["l2"]).abs(), b["e_d1"] + b["e_d2"]),
        "s0": _ratio(b["d0"].abs(), b["e_d0"]), "s1": _ratio(b["d1"].abs(), b["e_d1"]),
        "s2": _ratio(b["d2"].abs(), b["e_d2"]),
    }
    for n in DECISIONS:
        moves = torch.zeros_like(g5, dtype=torch.bool)
        for opt in OPTIONS[n]:
            alt = dict(d)
            alt[n] = torch.full_like(d[n], opt) if d[n].dtype != torch.bool else torch.full_like(d[n], bool(opt))
            a5, a6, _, _ = _orient_grad(b, alt)
            moves |= (a5 != g5) | (a6 != g6)
        ratios[n] = torch.where(moves, ratios[n], torch.full_like(ratios[n], math.inf))
    return dict(lp=lp, g5=g5, g6=g6, e5=e5, e6=e6, g8=g8, ratios=ratios, base=b, dec=d)


def _alternatives(o, H, W):
    """Every (g5, g6) an ambiguous pixel can take: all combinations of its ambiguous decisions' outcomes."""
    amb = torch.zeros_like(o["g5"], dtype=torch.bool)
    for k in DECISIONS:
        amb |= o["ratios"][k] < DECISION_SAFETY
    idx = torch.nonzero(amb).flatten()
    alts = {}
    for i in idx.tolist():
        b = {k: (v[i:i + 1] if isinstance(v, torch.Tensor) else v) for k, v in o["base"].items()}
        d = {k: v[i:i + 1] for k, v in o["dec"].items()}
        names = [k for k in DECISIONS if float(o["ratios"][k][i]) < DECISION_SAFETY]
        vals = []
        for combo in itertools.product(*[OPTIONS[k] for k in names]):
            dd = dict(d)
            for k, opt in zip(names, combo):
                dd[k] = torch.full_like(d[k], opt) if d[k].dtype != torch.bool else torch.full_like(d[k], bool(opt))
            a5, a6, e5, e6 = _orient_grad(b, dd)
            vals.append((float(a5), float(a6), float(e5), float(e6)))
        alts[divmod(i, W)] = (names, vals)
    return alts


# ------------------------------------------------------------------------------------------------ the replay
def _f64(a, device):
    if isinstance(a, np.ndarray):
        a = torch.from_numpy(np.ascontiguousarray(a))
    return a.to(device=device, dtype=torch.float64)


def replay(out, gt_image, gt_mask, gt_angle, gt_conf, lambdas, device=None, n_pixels=None, sum_w=None,
           consts=CONST32) -> dict:
    """out (10,H,W), gt_image (3,H,W), gt_mask (2,H,W), gt_angle (1,H,W), gt_conf (1,H,W): float32 arrays or tensors;
    lambdas = (l1, ssim, mask, orient).  The replay runs in float64 on `device` (default: out's).

    n_pixels / sum_w = (value, bound) override the image size and the sum of weights that scale the gradient (crops).
    consts = CONST64 replays a float64 evaluation of the reference (the eps, clamp and 1e-7 constants unrounded).

    Returns: sums {w, l1, ssim, mask, orient} and sums_scale; losses {total, Ll1, Lssim, Lmask, Lorient} and
    losses_scale; nan (Lorient was NaN); dL (10,H,W) and scale (10,H,W); ratios {decision: (H,W)}; alternatives
    {(y, x): (decision names, [(g5, g6, e5, e6), ...])}; ssim_map (3,H,W) and the per-pixel loss terms `terms`
    {name: (value (H,W), bound (H,W))}."""
    if device is None:
        device = out.device if isinstance(out, torch.Tensor) else torch.device("cpu")
    o, gi, gm, ga, gc = (_f64(a, device) for a in (out, gt_image, gt_mask, gt_angle, gt_conf))
    lam = [_f32(x) for x in lambdas]
    H, W = o.shape[1:]
    N = H * W if n_pixels is None else n_pixels
    m0, m1 = gm[0], gm[1]
    w = gc[0]
    if sum_w is None:
        sum_w = (float(w.sum()), float((1.0 + math.log2(max(N, 1))) * w.abs().sum()))
    wnd = window(device)
    # --- SSIM on image * gt_mask[1:], gt_image * gt_mask[1:]
    I, G = o[0:3], gi
    x, y = V(I) * V(m1.expand(3, H, W)), V(G) * V(m1.expand(3, H, W))
    mu1, mu2 = x.conv(wnd), y.conv(wnd)
    E11, E22, E12 = (x * x).conv(wnd), (y * y).conv(wnd), (x * y).conv(wnd)
    mu1_sq, mu2_sq, mu12 = mu1 * mu1, mu2 * mu2, mu1 * mu2
    s1, s2, s12 = E11 - mu1_sq, E22 - mu2_sq, E12 - mu12
    A1, A2 = 2.0 * mu12 + C1, 2.0 * s12 + C2
    B1, B2 = mu1_sq + mu2_sq + C1, s1 + s2 + C2
    BB = B1 * B2
    smap = A1 * A2 / BB
    D0 = 2.0 * mu2 * (A2 - A1) / BB - 2.0 * mu1 * smap * (B2 - B1) / BB
    D1 = -smap / B2
    D2 = 2.0 * A1 / BB
    s_ssim = V.c(-lam[1] / (3.0 * N), o[0])
    s_l1 = V.c(lam[0] / (3.0 * N), o[0])
    dS = D0.conv(wnd) + 2.0 * x * D1.conv(wnd) + y * D2.conv(wnd)
    sgn = torch.sign(I - G)
    g_img = s_ssim * dS * V(m1.expand(3, H, W)) + s_l1 * V(sgn * m1)
    # --- masks
    dmk = o[3:5] - gm
    dm_scale = lam[2] / (2.0 * N)
    g_mask = dm_scale * torch.sign(dmk)
    # --- orientation
    ori = _orient(o[5].reshape(-1), o[6].reshape(-1), o[8].reshape(-1), ga[0].reshape(-1), m0.reshape(-1),
                  w.reshape(-1), lam[3], sum_w[0], sum_w[1], consts)
    lp = ori["lp"]                        # already multiplied by m0 * w
    # --- per-pixel loss terms and the sums
    l1 = (I - G).abs() * m1
    terms = {"w": V(w), "l1": V(l1.sum(0), (2.0 * l1).sum(0)), "ssim": V(smap.v.sum(0), smap.e.sum(0)),
             "mask": V(dmk.abs().sum(0), dmk.abs().sum(0)),
             "orient": V(lp.v.reshape(H, W), lp.e.reshape(H, W))}
    sums, sums_scale = {}, {}
    for k in SUMS:
        sums[k], sums_scale[k] = _sum(terms[k], H * W)
    losses, losses_scale, nan = _finish(sums, sums_scale, N, lam)
    # --- gradient
    dL = torch.zeros(10, H, W, dtype=torch.float64, device=device)
    sc = torch.zeros_like(dL)
    dL[0:3], sc[0:3] = g_img.v, g_img.e
    dL[3:5], sc[3:5] = g_mask, g_mask.abs()
    if not nan:
        dL[5], sc[5] = ori["g5"].reshape(H, W), ori["e5"].reshape(H, W)
        dL[6], sc[6] = ori["g6"].reshape(H, W), ori["e6"].reshape(H, W)
        dL[8], sc[8] = ori["g8"].v.reshape(H, W), ori["g8"].e.reshape(H, W)
        ratios = {k: v.reshape(H, W) for k, v in ori["ratios"].items()}
        alts = _alternatives(ori, H, W)
    else:
        ratios = {k: torch.full((H, W), math.inf, dtype=torch.float64, device=device) for k in DECISIONS}
        alts = {}
    return dict(sums=sums, sums_scale=sums_scale, losses=losses, losses_scale=losses_scale, nan=nan, dL=dL, scale=sc,
                ratios=ratios, alternatives=alts, ssim_map=smap.v, terms=terms, sum_w=sum_w)


def _finish(sums, sums_scale, N, lam):
    """Loss values from the five sums (gh_image_loss's finalize; SRC/train_gaussians.py:126-140)."""
    n = float(N)
    with np.errstate(all="ignore"):
        Lo = np.float64(sums["orient"]) / np.float64(sums["w"])
    nan = bool(np.isnan(Lo))
    L = {"Ll1": sums["l1"] / (3 * n), "Lssim": 1.0 - sums["ssim"] / (3 * n), "Lmask": sums["mask"] / (2 * n),
         "Lorient": 0.0 if nan else float(Lo)}
    S = {"Ll1": sums_scale["l1"] / (3 * n) + abs(L["Ll1"]), "Lssim": 1.0 + sums_scale["ssim"] / (3 * n),
         "Lmask": sums_scale["mask"] / (2 * n) + abs(L["Lmask"]),
         "Lorient": 0.0 if nan else (sums_scale["orient"] + abs(Lo) * sums_scale["w"]) / abs(sums["w"]) + abs(Lo)}
    L["total"] = sum(l * L[k] for l, k in zip(lam, ("Ll1", "Lssim", "Lmask", "Lorient")))
    S["total"] = sum(abs(l) * (S[k] + abs(L[k])) for l, k in zip(lam, ("Ll1", "Lssim", "Lmask", "Lorient")))
    return L, S, nan


def replay_crop(inputs, lambdas, x0, y0, x1, y1, sum_w, device=None) -> dict:
    """The gradient, scale, ratios and alternatives of the rectangle [x0, x1) x [y0, y1) of the full-size inputs
    (out, gt_image, gt_mask, gt_angle, gt_conf as (C,H,W) tensors), replayed from the rectangle plus a HALO-pixel
    border (clipped at the image), with the global image size and sum_w = (sum of weights, its bound)."""
    H, W = inputs[0].shape[1:]
    X0, Y0, X1, Y1 = max(x0 - HALO, 0), max(y0 - HALO, 0), min(x1 + HALO, W), min(y1 + HALO, H)
    sub = [t[:, Y0:Y1, X0:X1] for t in inputs]
    r = replay(*sub, lambdas, device=device, n_pixels=H * W, sum_w=sum_w)
    sy, sx = slice(y0 - Y0, y1 - Y0), slice(x0 - X0, x1 - X0)
    alts = {(y + Y0, x + X0): v for (y, x), v in r["alternatives"].items()
            if y0 <= y + Y0 < y1 and x0 <= x + X0 < x1}
    return dict(dL=r["dL"][:, sy, sx], scale=r["scale"][:, sy, sx],
                ratios={k: v[sy, sx] for k, v in r["ratios"].items()}, alternatives=alts, origin=(y0, x0))


def chunked_sums(inputs, lambdas, rows=256, device=None) -> dict:
    """The five sums, their bounds and the losses of a full-size image, replayed in bands of `rows` rows (each with a
    5-row halo for the SSIM window).  Returns sums, sums_scale, losses, losses_scale, nan."""
    H, W = inputs[0].shape[1:]
    N = H * W
    gc = inputs[4]
    sw = float(gc.double().sum())
    sw_e = float((1.0 + math.log2(N)) * gc.double().abs().sum())
    sums = {k: 0.0 for k in SUMS}
    scal = {k: 0.0 for k in SUMS}
    for r0 in range(0, H, rows):
        r1 = min(r0 + rows, H)
        Y0, Y1 = max(r0 - R, 0), min(r1 + R, H)
        sub = [t[:, Y0:Y1] for t in inputs]
        r = replay(*sub, lambdas, device=device, n_pixels=N, sum_w=(sw, sw_e))
        own = slice(r0 - Y0, r1 - Y0)
        for k in SUMS:
            t = r["terms"][k]
            sums[k] += float(t.v[own].sum())
            scal[k] += float(t.e[own].sum() + (1.0 + math.log2(N)) * t.v[own].abs().sum())
    losses, losses_scale, nan = _finish(sums, scal, N, [_f32(x) for x in lambdas])
    return dict(sums=sums, sums_scale=scal, losses=losses, losses_scale=losses_scale, nan=nan)


# ------------------------------------------------------------------------------------------------ edge scenes
# (c5, c6, conf, gt_angle, gt_mask[0], gt_orient_conf) of pixels that sit on a branch of the orientation path:
# c6 = 0 gives t = 0 and ang = 0.5 exactly, and with gt_angle 0, 0.5, 1 the ties l0 = l1, d0 = 0 and l0 = l2; c5 = 0
# and |c6| = 1 clamp with a zero derivative, |c5| = 0.01 clamp with a non-zero one; (3, 4) has an exact norm; a zero
# direction with conf > 0 takes the 1e12 eps gradient; norms 1e-13 (eps branch), exactly float32(1e-12) (the nrm >= eps
# branch, with the same value) and 2e-12; the last is a background pixel (channels 5..8 zero) under gt_mask[0] = 1.
ORIENT_SPECIALS = (
    [(c5, 0.0, 0.5, g, 1.0, 0.5) for c5 in (1.0, -1.0, 0.0, -0.0) for g in (0.0, 0.5, 1.0)]
    + [(0.0, 1.0, 0.5, 0.3, 1.0, 0.5), (0.0, -1.0, 0.5, 0.3, 1.0, 0.5), (0.01, 1.0, 0.6, 0.2, 1.0, 0.7),
       (-0.01, -1.0, 0.6, 0.8, 1.0, 0.7), (0.01, -1.0, 0.4, 0.6, 1.0, 0.3), (3.0, 4.0, 0.5, 0.1, 1.0, 0.5),
       (-3.0, 4.0, 0.5, 0.9, 1.0, 0.5), (3.0, -4.0, 0.5, 0.4, 1.0, 0.5), (0.0, 0.0, 0.7, 0.2, 1.0, 0.6),
       (0.6e-13, 0.8e-13, 0.7, 0.2, 1.0, 0.6), (1e-12, 0.0, 0.7, 0.3, 1.0, 0.6), (-2e-12, 0.0, 0.7, 0.6, 1.0, 0.6),
       (1.2e-12, 1.6e-12, 0.7, 0.7, 1.0, 0.6), (0.0, 0.0, 0.0, 0.3, 1.0, 0.5)])


def edge_scene(W: int, H: int, seed: int = 0, specials: bool = True):
    """Float32 (render, gt_image, gt_mask, gt_angle, gt_conf) on the CPU: random maps like a training view (binary and
    fractional masks, random directions) with, when `specials`, the pixels of ORIENT_SPECIALS spread over the image
    (corners first), columns where the render equals gt_image and rows where the mask channels equal gt_mask (masks 0, 1
    and fractional), and, where the image is large enough, a 13x13 block with gt_mask[1] = 0 and a 15x15 block of
    constant image and target (sigma = 0: b2 at its C2 floor)."""
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.rand(*s, generator=g)   # noqa: E731
    out = torch.empty(10, H, W)
    out[0:3] = r(3, H, W)
    out[3:5] = r(2, H, W)
    out[5:8] = r(3, H, W) * 2 - 1
    out[8] = r(H, W) * 0.9 + 0.05
    out[9] = r(H, W) * 3
    gi = r(3, H, W)
    u = r(2, H, W)
    gm = torch.where(u < 0.3, 0.0, torch.where(u < 0.65, 1.0, r(2, H, W)))
    ga = r(1, H, W)
    gc = r(1, H, W)
    if specials:
        n = H * W
        corners = [0, W - 1, (H - 1) * W, n - 1]
        rest = torch.randperm(n, generator=g).tolist()
        where = list(dict.fromkeys(corners + rest))[:min(n, len(ORIENT_SPECIALS))]
        for i, (c5, c6, conf, ang, m0, w) in zip(where, ORIENT_SPECIALS):
            y, x = divmod(i, W)
            out[5, y, x], out[6, y, x], out[8, y, x] = c5, c6, conf
            ga[0, y, x], gm[0, y, x], gc[0, y, x] = ang, m0, w
            if conf == 0.0:
                out[5:9, y, x] = 0.0
        out[0:3, :, 1::3] = gi[:, :, 1::3]                # I == G
        out[3:5, ::2] = gm[:, ::2]                        # mask == gt_mask
        if H >= 20 and W >= 20:
            gm[1, 2:15, 3:16] = 0.0
        if H >= 30 and W >= 35:
            out[0:3, 14:29, 18:33] = torch.tensor([0.25, 0.5, 0.75])[:, None, None]
            gi[:, 14:29, 18:33] = torch.tensor([0.5, 0.125, 0.75])[:, None, None]
            gm[1, 14:29, 18:33] = 1.0
    return out, gi, gm, ga, gc
