"""TEST INFRASTRUCTURE ONLY -- the float64 oracle of the mesh rasterizer (csrc/gh_mesh_raster.cu, DESIGN §24), and a
numpy restatement of the scalp script's visibility logic (extract_non_visible_head_scalp.py:51-93).

`raster64(verts, faces, K, R, t, H, W)` enumerates every (face, pixel) pair near a face's projection and gives, in
float64 (torch, on any device):
  * W (n,3) the exact edge functions and A the exact doubled area, each with a float32 error bound E derived from the
    operation order of gh_mesh_math.h (gh_raster_setup, gh_raster_edges, gh_raster_pixel) -- no calibrated factor:
      u = 2^-24, gamma_n = n u / (1 - n u);  x_cam = fma(R0, X, fma(R1, Y, fma(R2, Z, t0))) within gamma_3 (|R0 X| +
      |R1 Y| + |R2 Z| + |t0|);  u = fma(fx, x/z, cx) from the propagated x, z errors plus one rounding per division
      and fma;  w = fma(a, b, -(c d)) with a, b, c, d differences of screen coordinates: the vertex errors through the
      bilinear form (|a| eb + |b| ea + ea eb + |c| ed + |d| ec + ec ed) plus gamma_4 ((|a| + ea)(|b| + eb) + (|c| +
      ec)(|d| + ed)); the depth z = A / S, S = sum w_k / z_k, within [(|A| - E_A) / (|S| + E_S), (|A| + E_A) /
      (|S| - E_S)] (1 -+ u), E_S from the w and 1/z bounds and gamma_3 for the two fmas and the product;
    float64's own rounding is added as gamma_n in 2^-53 on the same magnitudes;
  * cert / poss: the pair is covered for every float32 result within the bounds / for some;
  * per pixel: `decided` (exactly one admissible answer), `answer` where decided, and the admissible answers: -1 iff
    no pair is certainly covered, a face iff possibly covered and its lowest depth is not above the highest depth of a
    certainly covered face.
"""
from __future__ import annotations

import math

import numpy as np
import torch

U = 2.0 ** -24
D = 2.0 ** -53


def gam(n):
    return n * U / (1 - n * U)


def gd(n):
    return n * D / (1 - n * D)


def _bil(a, ea, b, eb, c, ec, d, ed):
    """Bound on |(a b - c d) computed in float32 from inputs within ea.. of a.. - (a b - c d)|."""
    ab = (a.abs() + ea) * (b.abs() + eb)
    cd = (c.abs() + ec) * (d.abs() + ed)
    return (a.abs() * eb + b.abs() * ea + ea * eb + c.abs() * ed + d.abs() * ec + ec * ed + gam(4) * (ab + cd)
            + gd(6) * (ab + cd))


def vertices64(verts, K, R, t):
    """Exact camera coordinates and screen positions of float32 vertices, with the float32 errors of the setup."""
    X = verts.double()
    R, t, K = R.double(), t.double(), K.double()
    terms = X[:, None, :] * R[None]                              # (V, 3 rows, 3)
    cam = terms.sum(-1) + t
    mag = terms.abs().sum(-1) + t.abs()
    e = (gam(3) + gd(4)) * mag
    x, y, z = cam.unbind(-1)
    ex, ey, ez = e.unbind(-1)
    fx, fy, cx, cy = K[0, 0], K[1, 1], K[0, 2], K[1, 2]
    out = {"z": z, "ez": ez}
    for name, p, ep, f, c in (("u", x, ex, fx, cx), ("v", y, ey, fy, cy)):
        s = p / z
        den = z.abs() - ez
        es = torch.where(den > 0, (ep + s.abs() * ez) / den.clamp_min(1e-300), torch.full_like(s, math.inf))
        es = es + U * (s.abs() + es)
        out[name] = f * s + c
        out["e" + name] = f.abs() * es + (U + gd(3)) * (f.abs() * (s.abs() + es) + c.abs())
    iz = 1.0 / z
    den = z.abs() - ez
    eiz = torch.where(den > 0, ez / (z.abs() * den.clamp_min(1e-300)), torch.full_like(z, math.inf))
    out["iz"], out["eiz"] = iz, eiz + (U + gd(1)) * (iz.abs() + eiz)
    out["finite"] = torch.isfinite(X).all(-1)
    return out


def raster64(verts, faces, K, R, t, H, W, device="cpu", margin=2):
    """One view.  verts (V,3) float32, faces (F,3) int32 (all in range), K/R (3,3), t (3): numpy or torch."""
    tt = lambda a: torch.as_tensor(np.asarray(a) if not torch.is_tensor(a) else a, device=device)  # noqa: E731
    verts, faces, K, R, t = tt(verts), tt(faces).long(), tt(K), tt(R), tt(t)
    F = faces.shape[0]
    vx = vertices64(verts, K, R, t)
    g = {k: v[faces] for k, v in vx.items()}                     # (F, 3) each
    finite = g["finite"].all(1)
    front_cert = (g["z"] > g["ez"]).all(1) & finite
    front_poss = (g["z"] > -g["ez"]).all(1) & finite
    u, v, eu, ev = (torch.nan_to_num(g[k], nan=0.0, posinf=0.0, neginf=0.0) for k in ("u", "v", "eu", "ev"))
    A = (u[:, 1] - u[:, 0]) * (v[:, 2] - v[:, 0]) - (v[:, 1] - v[:, 0]) * (u[:, 2] - u[:, 0])
    EA = _bil(u[:, 1] - u[:, 0], eu[:, 1] + eu[:, 0], v[:, 2] - v[:, 0], ev[:, 2] + ev[:, 0],
              v[:, 1] - v[:, 0], ev[:, 1] + ev[:, 0], u[:, 2] - u[:, 0], eu[:, 2] + eu[:, 0])
    drawn_cert = front_cert & (A.abs() > EA) & (eu.amax(1) < 1) & (ev.amax(1) < 1)
    drawn_poss = front_poss
    # candidate pixels: the exact box of the projection plus `margin` pixels (the errors are far below a pixel)
    big = 4.0 * max(H, W)
    j0 = torch.floor((u - eu).amin(1).clamp(-big, big)) - margin
    j1 = torch.ceil((u + eu).amax(1).clamp(-big, big)) + margin
    i0 = torch.floor((v - ev).amin(1).clamp(-big, big)) - margin
    i1 = torch.ceil((v + ev).amax(1).clamp(-big, big)) + margin
    j0, i0 = j0.clamp(0, W - 1).long(), i0.clamp(0, H - 1).long()
    j1, i1 = j1.clamp(-1, W - 1).long(), i1.clamp(-1, H - 1).long()
    nj, ni = (j1 - j0 + 1).clamp_min(0), (i1 - i0 + 1).clamp_min(0)
    n = torch.where(drawn_poss, nj * ni, torch.zeros_like(nj))
    face = torch.repeat_interleave(torch.arange(F, device=device), n)
    off = torch.cumsum(n, 0) - n
    local = torch.arange(face.shape[0], device=device) - off[face]
    row = i0[face] + local // nj[face]
    col = j0[face] + local % nj[face]
    px, py = col.double() + 0.5, row.double() + 0.5
    uf, vf, euf, evf = u[face], v[face], eu[face], ev[face]
    Wk, EW = [], []
    for k in range(3):
        k1, k2 = (k + 1) % 3, (k + 2) % 3
        a, ea = uf[:, k2] - uf[:, k1], euf[:, k2] + euf[:, k1]
        b, eb = py - vf[:, k1], evf[:, k1]
        c, ec = vf[:, k2] - vf[:, k1], evf[:, k2] + evf[:, k1]
        d, ed = px - uf[:, k1], euf[:, k1]
        Wk.append(a * b - c * d)
        EW.append(_bil(a, ea, b, eb, c, ec, d, ed))
    Wk, EW = torch.stack(Wk, 1), torch.stack(EW, 1)
    Af, EAf = A[face], EA[face]
    sA = torch.sign(Af)
    dec = Wk.abs() > EW
    sW = torch.sign(Wk)
    area_dec = Af.abs() > EAf
    cert = drawn_cert[face] & (dec & (sW == sA[:, None])).all(1)
    pos_dec, neg_dec = (dec & (sW > 0)).any(1), (dec & (sW < 0)).any(1)
    against_area = (dec & (sW != sA[:, None])).any(1)
    poss = drawn_poss[face] & ~(pos_dec & neg_dec) & ~(area_dec & against_area)
    izf, eizf = g["iz"][face], g["eiz"][face]
    S = (Wk * izf).sum(1)
    ES = (Wk.abs() * eizf + izf.abs() * EW + EW * eizf).sum(1) + \
        (gam(3) + gd(6)) * ((Wk.abs() + EW) * (izf.abs() + eizf)).sum(1)
    z = Af / S
    lo_den, hi_den = S.abs() + ES, S.abs() - ES
    z_lo = ((Af.abs() - EAf).clamp_min(0) / lo_den) * (1 - U) * (1 - gd(4))
    z_hi = torch.where(hi_den > 0, (Af.abs() + EAf) / hi_den.clamp_min(1e-300) * (1 + U) * (1 + gd(4)),
                       torch.full_like(z, math.inf))
    # per pixel
    pix = row * W + col
    HW = H * W
    n_cert = torch.zeros(HW, dtype=torch.long, device=device).index_add_(0, pix, cert.long())
    minhi = torch.full((HW,), math.inf, dtype=torch.float64, device=device)
    minhi.scatter_reduce_(0, pix[cert], z_hi[cert], reduce="amin")
    adm = poss & (z_lo <= minhi[pix])
    neg_adm = n_cert == 0
    n_adm = torch.zeros(HW, dtype=torch.long, device=device).index_add_(0, pix, adm.long()) + neg_adm.long()
    decided = n_adm == 1
    answer = torch.full((HW,), -1, dtype=torch.long, device=device)
    win = adm & decided[pix]
    answer[pix[win]] = face[win]
    return {"face": face, "row": row, "col": col, "pix": pix, "W": Wk, "EW": EW, "A": Af, "EA": EAf, "z": z,
            "z_lo": z_lo, "z_hi": z_hi, "cert": cert, "poss": poss, "adm": adm, "neg_adm": neg_adm.view(H, W),
            "decided": decided.view(H, W), "answer": answer.view(H, W), "drawn_cert": drawn_cert,
            "front_poss": front_poss, "front_cert": front_cert}


def admissible(o, p2f, F):
    """bool (H, W): the kernel's pix_to_face (torch, on the oracle's device) is an admissible answer at each pixel."""
    H, W = p2f.shape
    p = p2f.reshape(-1).long()
    ok = (p < 0) & o["neg_adm"].reshape(-1)
    keys = torch.sort(o["pix"][o["adm"]] * (F + 1) + o["face"][o["adm"]])[0]
    q = torch.arange(H * W, device=p.device) * (F + 1) + p
    if keys.numel():
        hit = keys[torch.searchsorted(keys, q).clamp_max(keys.numel() - 1)] == q
    else:
        hit = torch.zeros_like(ok)
    return (ok | ((p >= 0) & hit)).view(H, W)


def face_sets(o, head, F):
    """Per view: the faces every admissible outcome shows (lo) and those some outcome may show (hi), in the plain and
    the head-masked variant, and whether -1 certainly occurs in each.  head: bool (H, W) torch."""
    h = head.reshape(-1)
    dec = o["decided"].reshape(-1)
    ans = o["answer"].reshape(-1)
    adm_pix, adm_face = o["pix"][o["adm"]], o["face"][o["adm"]]
    out = {}
    for name, m in (("plain", torch.ones_like(h)), ("head", h)):
        lo = torch.zeros(F, dtype=torch.bool, device=h.device)
        sel = dec & (ans >= 0) & m
        lo[ans[sel]] = True
        hi = lo.clone()
        und = ~dec[adm_pix] & m[adm_pix]
        hi[adm_face[und]] = True
        out[name] = (lo, hi, bool(((dec & (ans < 0)) | ~m).any()))
    return out


# ------------------------------------------------------------------------------------ the script's visibility logic
def script_visibility(pix_to_face, head, faces, V):
    """extract_non_visible_head_scalp.py:51-93 restated in numpy: pix_to_face (B,H,W) int, head (B,H,W) bool, faces
    (F,3) -> (vis_mask bool (V,), vis_maps float32 (V,), vis_maps_head float32 (V,))."""
    B = pix_to_face.shape[0]
    vs, vhs = [], []
    for b in range(B):
        p = pix_to_face[b]
        ph = np.where(head[b], p, -1)
        v = np.zeros(V, np.float32)
        vh = np.zeros(V, np.float32)
        v[np.unique(faces[np.unique(p)[1:]])] = 1.0
        vh[np.unique(faces[np.unique(ph)[1:]])] = 1.0
        vs.append(v)
        vhs.append(vh)
    vis_maps = np.stack(vs).sum(0).astype(np.float32)
    vis_maps_head = np.stack(vhs).sum(0).astype(np.float32)
    with np.errstate(invalid="ignore", divide="ignore"):
        prob_hair = np.float32(1) - vis_maps_head / vis_maps
    vis_mask = (prob_hair > 0.5) | (vis_maps / np.float32(B) < 0.1)
    return vis_mask, vis_maps, vis_maps_head


# ------------------------------------------------------------------------------------------------------- cameras
def look_at(eye, target, up=(0.0, 0.0, 1.0)):
    """OpenCV world-to-camera (R, t): z forward towards target, x right, y down."""
    eye, target, up = (np.asarray(a, np.float64) for a in (eye, target, up))
    z = target - eye
    z /= np.linalg.norm(z)
    x = np.cross(z, up)
    if np.linalg.norm(x) < 1e-9:
        x = np.cross(z, [1.0, 0.0, 0.0])
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    R = np.stack([x, y, z])
    return R, -R @ eye


def sphere_cameras(B, H, W, seed, radius=0.45, f_scale=1.3, jitter=0.01):
    """B cameras on a sphere (Fibonacci directions, jittered aim and focal length) looking at the origin: K, R, t
    float32 (B,3,3), (B,3,3), (B,3)."""
    rng = np.random.default_rng(seed)
    Ks, Rs, ts = [], [], []
    for b in range(B):
        zc = 1 - 2 * (b + 0.5) / B
        phi = b * math.pi * (3 - math.sqrt(5)) + rng.uniform(0, 0.3)
        d = np.array([math.sqrt(1 - zc * zc) * math.cos(phi), math.sqrt(1 - zc * zc) * math.sin(phi), zc])
        R, t = look_at(d * radius * rng.uniform(0.9, 1.1), rng.normal(0, jitter, 3))
        f = f_scale * max(H, W) * rng.uniform(0.9, 1.1)
        Ks.append([[f, 0, W / 2 + rng.uniform(-3, 3)], [0, f, H / 2 + rng.uniform(-3, 3)], [0, 0, 1]])
        Rs.append(R)
        ts.append(t)
    return tuple(np.asarray(a, np.float32) for a in (Ks, Rs, ts))
