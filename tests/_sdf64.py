"""TEST INFRASTRUCTURE ONLY -- the float64 oracle of the mesh signed distance (gh_sdf_query, gaussianhaircut_b200.mesh)
and of the FLAME-intersection filter, brute force in numpy, with first-order bounds of the kernels' float32 evaluation.

Per (point p, face f), with A = a - p, B = b - p, C = c - p, n = ab x ac and u = 2^-24 (all in float64):
    d_f      distance from p to the triangle: the smallest edge-segment distance and, when p's projection lies in the
             face (B x C, C x A, A x B all on n's side), the plane distance |A . n| / |n|; a triangle with n = 0 is its
             edges, an edge of length 0 its vertex
    Omega_f  2 atan2(A . (B x C), |A||B||C| + (A.B)|C| + (A.C)|B| + (B.C)|A|)
and per point d = min_f d_f, w = sum_f Omega_f / 4 pi, sdf = d if w > 0.5 else -d.

Bounds (gaussianhaircut_b200/csrc/gh_mesh_math.h's operation order; one rounding counted per multiply and per add, so a
contracted FMA is covered; R = |A| + |B| + |C|, kappa = |ab||ac| / |n| >= 1):
    edge segment  the vertex difference X and the edge E carry u relative, 1 / |E|^2 6 u, X . E 5 u |X||E|: t is off by
                  5 u |X| / |E| + 7 u, which moves the distance by at most 5 u |X| + 7 u |E| (t* is the minimiser);
                  Q = X + t E adds 2 u |X| + 3 u |E|, |Q|^2 and the final square root 2 u |X|:  <= SEG u R, SEG = 19
    plane         n is off by 5 u |ab||ac|, A . n by 4 u |A||n| + 5 u |A||ab||ac|, 1 / |n|^2 and the square root by
                  4 u:  <= u R (PL0 + PL1 kappa), PL0 = 8, PL1 = 10 -- counted wherever the face branch can be taken
    face test     T = (X x Y) . n is off by dT = u |X||Y||n| (12 + 6 kappa); where |T| <= dT for one of the three
                  tests and none is certainly negative the kernel may take either branch, and the bound also holds the
                  difference between the two exact branch values
    record        the float32 record (record32, bit-identical to gh_sdf_record) decides which branches exist: a face
                  whose float32 1 / |n|^2 is 0 is only its edges in the kernel, an edge whose 1 / |E|^2 is 0 only its
                  vertex; the exact distance of that restricted formula minus d_f is added to the bound
    solid angle   num is off by NUM u |A||B||C|, den by DEN u |A||B||C| (NUM = 10, DEN = 50), atan2f by 2 ulp (CUDA's
                  documented maximum, 4 u |Omega| for Omega = 2 atan2): dOmega = 2 (|den| dnum + |num| dden) /
                  (num^2 + den^2) + 4 u |Omega|, or 4 pi + 2^-20 when (num, den) is within (dnum, dden) of the branch cut
                  (den < 0, |num| <= dnum) or of the origin.  The sum is in double: F 2^-50 more.
So the kernel's d lies in [min_f (d_f - e_f), min_f (d_f + e_f)] and |w_kernel - w| <= sum_f dOmega_f / 4 pi + F 2^-50
(+ the float32 rounding of the output).  The sign is decided where |w - 0.5| and d exceed their bounds.

Filter (filter_flame_intersections.py:88, 104-119): the corners in float64 from the same float32 inputs; a float32
corner is off by at most CORNER u (90 sigma + 2 max|xyz|), sigma = 3 max(scaling): build_rotation's normalised
quaternion 4.5 u, R entries 23 u, M = S R 25 u sigma, v @ M + xyz with the float32 icosahedron (u each) and a 3-term sum.
Moving a corner by e moves w by at most e sum_f perimeter_f / (4 pi d_f^2).
"""
from __future__ import annotations

import math
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np

U = 2.0 ** -24
SEG, PL0, PL1, T0, T1 = 19.0, 8.0, 10.0, 12.0, 6.0
NUM, DEN = 10.0, 50.0
CORNER_SIGMA, CORNER_XYZ = 90.0, 2.0


def record32(verts: np.ndarray, faces: np.ndarray) -> np.ndarray:
    """(F,28) float32: gh_sdf_record of every face, bit for bit (numpy rounds every float32 operation on its own)."""
    v = verts.astype(np.float32)
    a, b, c = v[faces[:, 0]], v[faces[:, 1]], v[faces[:, 2]]
    ab, bc, ca = b - a, c - b, a - c
    n = np.stack([ca[:, 1] * ab[:, 2] - ca[:, 2] * ab[:, 1], ca[:, 2] * ab[:, 0] - ca[:, 0] * ab[:, 2],
                  ca[:, 0] * ab[:, 1] - ca[:, 1] * ab[:, 0]], 1)

    def rcp(x):
        nn = (x[:, 0] * x[:, 0] + x[:, 1] * x[:, 1]) + x[:, 2] * x[:, 2]
        with np.errstate(divide="ignore", over="ignore", invalid="ignore"):
            r = np.float32(1) / nn
        return np.where((r > 0) & (r < np.inf), r, np.float32(0)).astype(np.float32)

    z = np.zeros(len(faces), np.float32)
    cols = [a, rcp(n)[:, None], b, rcp(ab)[:, None], c, rcp(bc)[:, None], ab, rcp(ca)[:, None], bc, z[:, None], ca,
            z[:, None], n, z[:, None]]
    return np.concatenate(cols, 1).astype(np.float32)


def _dot(x, y):
    return x[..., 0] * y[..., 0] + x[..., 1] * y[..., 1] + x[..., 2] * y[..., 2]


def _norm(x):
    return np.sqrt(_dot(x, x))


def _seg(X, E, ok=None):
    """Distance from the origin to {X + t E, t in [0, 1]}; where `ok` is False, to X alone."""
    ee = _dot(E, E)
    with np.errstate(divide="ignore", invalid="ignore"):
        t = np.where(ee > 0, np.clip(-_dot(X, E) / np.where(ee > 0, ee, 1), 0, 1), 0)
    if ok is not None:
        t = np.where(ok, t, 0)
    return _norm(X + t[..., None] * E)


class Mesh64:
    """A mesh for the oracle: float64 vertex triples and the float32 record flags of the kernel."""

    def __init__(self, verts: np.ndarray, faces: np.ndarray):
        faces = np.asarray(faces, np.int64)
        v = np.asarray(verts, np.float32).astype(np.float64)
        self.F = len(faces)
        self.a, self.b, self.c = v[faces[:, 0]], v[faces[:, 1]], v[faces[:, 2]]
        self.ab, self.bc, self.ca = self.b - self.a, self.c - self.b, self.a - self.c
        self.n = np.cross(self.ab, self.c - self.a)
        self.nn = _norm(self.n)
        with np.errstate(divide="ignore", invalid="ignore"):
            self.kappa = np.where(self.nn > 0, _norm(self.ab) * _norm(self.ca) / self.nn, np.inf)
        self.perimeter = _norm(self.ab) + _norm(self.bc) + _norm(self.ca)
        rec = record32(verts, faces)
        self.face32 = rec[:, 3] > 0                     # the kernel's face branch exists
        self.edge32 = rec[:, [7, 11, 15]] > 0           # ab, bc, ca: not reduced to their vertex


def pairs(p: np.ndarray, m: Mesh64, face=None) -> dict:
    """d, omega, e (the distance bound) and domega: per (point, face) (n, F) for every face, or with `face` (n,) per
    pair (p[i], face[i])."""
    p = np.asarray(p, np.float64)
    if face is None:
        p, sl = p[:, None, :], (None, slice(None))
    else:
        sl = face
    a, b, c = m.a[sl], m.b[sl], m.c[sl]
    ab, bc, ca, n = m.ab[sl], m.bc[sl], m.ca[sl], m.n[sl]
    nn, kappa = m.nn[sl], m.kappa[sl]
    A, B, C = a - p, b - p, c - p
    la, lb, lc = _norm(A), _norm(B), _norm(C)
    R = la + lb + lc
    bxc, cxa, axb = np.cross(B, C), np.cross(C, A), np.cross(A, B)
    T = np.stack([_dot(bxc, n), _dot(cxa, n), _dot(axb, n)], -1)
    dT = U * np.stack([lb * lc, lc * la, la * lb], -1) * (nn * (T0 + T1 * np.minimum(kappa, 1e300)))[..., None]
    edges = np.minimum(np.minimum(_seg(A, ab), _seg(B, bc)), _seg(C, ca))
    e32 = m.edge32[sl]
    edges_k = np.minimum(np.minimum(_seg(A, ab, e32[..., 0]), _seg(B, bc, e32[..., 1])), _seg(C, ca, e32[..., 2]))
    with np.errstate(divide="ignore", invalid="ignore"):
        plane = np.where(nn > 0, np.abs(_dot(A, n)) / np.where(nn > 0, nn, 1), np.inf)
    inside = (nn > 0) & (T >= 0).all(-1)
    d = np.where(inside, np.minimum(edges, plane), edges)
    face32 = np.broadcast_to(m.face32[sl], d.shape)
    certain_in = face32 & (T > dT).all(-1)
    certain_out = ~face32 | (T < -dT).any(-1)
    in_k, out_k = np.minimum(edges_k, plane), edges_k          # the kernel's two branches, exactly
    dev = np.where(certain_in, np.abs(in_k - d), np.where(certain_out, np.abs(out_k - d),
                                                            np.maximum(np.abs(in_k - d), np.abs(out_k - d))))
    with np.errstate(invalid="ignore"):
        e = SEG * U * R + dev + np.where(certain_out, 0.0, U * R * (PL0 + PL1 * kappa))
    # solid angle
    num = _dot(A, bxc)
    den = la * lb * lc + _dot(A, B) * lc + _dot(A, C) * lb + _dot(B, C) * la
    omega = 2.0 * np.arctan2(num, den)
    s3 = la * lb * lc
    dnum, dden = NUM * U * s3, DEN * U * s3
    with np.errstate(divide="ignore", invalid="ignore"):
        dom = 2.0 * (np.abs(den) * dnum + np.abs(num) * dden) / (num * num + den * den) + 4 * U * np.abs(omega)
    cut = ((den < dden) & (np.abs(num) <= dnum)) | ((np.abs(num) <= dnum) & (np.abs(den) <= dden))
    dom = np.where(cut | ~np.isfinite(dom), 4 * math.pi + 2.0 ** -20, dom)     # float32 2 atan2 <= 2 pi + 2^-21
    return {"d": d, "omega": omega, "e": e, "domega": dom}


def _query_chunk(p, m, want_grad):
    q = pairs(p, m)
    d, e = q["d"], q["e"]
    out = {"d": d.min(1), "lo": (d - e).min(1), "hi": (d + e).min(1),
           "w": q["omega"].sum(1) / (4 * math.pi), "ew": q["domega"].sum(1) / (4 * math.pi) + m.F * 2.0 ** -50}
    if want_grad:
        with np.errstate(divide="ignore"):
            out["wgrad"] = (m.perimeter[None] / (d * d)).sum(1) / (4 * math.pi)
    return out


def query64(points: np.ndarray, verts: np.ndarray, faces: np.ndarray, want_grad: bool = False, chunk: int = 0) -> dict:
    """Per point (rows with a non-finite coordinate get NaN): d, lo, hi (the kernel's d lies in [lo, hi]), w, ew (the
    bound of |w_kernel - w|), sdf, and with want_grad the bound of |dw/dp|.  Brute force over every face, chunks of
    points in threads."""
    m = Mesh64(verts, faces)
    p = np.asarray(points, np.float32).astype(np.float64)
    fin = np.isfinite(p).all(1)
    idx = np.nonzero(fin)[0]
    chunk = chunk or max(1, min(256, 2_000_000 // max(1, m.F)))
    parts = [idx[i:i + chunk] for i in range(0, len(idx), chunk)]
    with ThreadPoolExecutor(max_workers=min(32, os.cpu_count() or 1)) as ex:
        res = list(ex.map(lambda ix: _query_chunk(p[ix], m, want_grad), parts))
    keys = ["d", "lo", "hi", "w", "ew"] + (["wgrad"] if want_grad else [])
    out = {k: np.full(len(p), np.nan) for k in keys}
    for ix, r in zip(parts, res):
        for k in keys:
            out[k][ix] = r[k]
    out["sdf"] = np.where(out["w"] > 0.5, out["d"], -out["d"])
    return out


# ------------------------------------------------------------------------------------------------------- the filter
def icosahedron64() -> np.ndarray:
    t = (1.0 + math.sqrt(5.0)) / 2.0
    v = np.array([[-1, t, 0], [1, t, 0], [-1, -t, 0], [1, -t, 0], [0, -1, t], [0, 1, t], [0, -1, -t], [0, 1, -t],
                  [t, 0, -1], [t, 0, 1], [-t, 0, -1], [-t, 0, 1]], np.float64)
    return v / np.linalg.norm(v, axis=1, keepdims=True)


def flame_corners64(xyz, scaling, rotation) -> np.ndarray:
    """(P,12,3): build_scaling_rotation(scaling * 3, rotation) and v @ M + xyz in float64 (script lines 88, 108)."""
    xyz, s, r = (np.asarray(x, np.float32).astype(np.float64) for x in (xyz, scaling, rotation))
    q = r / np.sqrt((r * r).sum(1))[:, None]
    w, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    R = np.empty((len(q), 3, 3))
    R[:, 0, 0] = 1 - 2 * (y * y + z * z)
    R[:, 1, 0] = 2 * (x * y - w * z)
    R[:, 2, 0] = 2 * (x * z + w * y)
    R[:, 0, 1] = 2 * (x * y + w * z)
    R[:, 1, 1] = 1 - 2 * (x * x + z * z)
    R[:, 2, 1] = 2 * (y * z - w * x)
    R[:, 0, 2] = 2 * (x * z - w * y)
    R[:, 1, 2] = 2 * (y * z + w * x)
    R[:, 2, 2] = 1 - 2 * (x * x + y * y)
    M = (s * 3)[:, :, None] * R                   # S @ R
    return np.einsum("vi,pij->pvj", icosahedron64(), M) + xyz[:, None, :]


def corner_bound(xyz, scaling) -> np.ndarray:
    """(P,): the bound of |float32 corner - float64 corner| for every corner of each Gaussian."""
    xyz, s = np.asarray(xyz, np.float64), np.asarray(scaling, np.float64)
    return U * (CORNER_SIGMA * 3 * s.max(1) + CORNER_XYZ * np.abs(xyz).max(1))


def flame_filter_keep64(xyz, scaling, rotation, label, verts, faces) -> dict:
    """Script lines 88, 104-119 in float64: keep (P,) bool, and `clear` (P,) bool -- every corner of the Gaussian lies
    farther from the surface, and its winding number farther from 0.5, than the corner and SDF bounds, so the float32
    pipeline must decide it the same way (Gaussians with label <= 0.5 are kept either way and always clear)."""
    corners = flame_corners64(xyz, scaling, rotation)
    P = corners.shape[0]
    q = query64(corners.reshape(-1, 3), verts, faces, want_grad=True)
    ec = np.repeat(corner_bound(xyz, scaling), 12)
    clear_d = q["lo"] > ec                         # d > e_c + (d - lo): the perturbed corner is off the surface too
    clear_w = np.abs(q["w"] - 0.5) > q["ew"] + ec * q["wgrad"]
    outside = (q["sdf"] < 0).reshape(P, 12).all(1)
    low = np.asarray(label, np.float32).reshape(P) <= np.float32(0.5)
    clear = (clear_d & clear_w).reshape(P, 12).all(1) | low
    return {"keep": outside | low, "clear": clear, "corners": corners}
