"""TEST INFRASTRUCTURE ONLY -- seeded meshes, query sets and Gaussian scenes for the mesh signed distance
(tests/test_sdf_cpu.py, tests/test_gpu_sdf.py).  Sizes are in metres, like a FLAME head (~0.1 m across).

Meshes: (verts (V,3) float32, faces (F,3) int32), faces counter-clockwise seen from outside.
    icosphere     a level-3 subdivided icosahedron (1 280 faces), radius 0.1
    head          a deformed ellipsoid: 69 latitude rings of 72 vertices and two pole fans (9 936 faces)
    head_holes    the head with five caps removed (eyes, mouth, neck, a crown hole): an open mesh
    degenerate    a level-2 icosphere plus duplicated faces, point, segment and collinear triangles
    big           a level-6 icosphere (81 920 faces)
"""
from __future__ import annotations

import math
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def icosphere(level: int, radius: float = 0.1):
    t = (1.0 + math.sqrt(5.0)) / 2.0
    v = [[-1, t, 0], [1, t, 0], [-1, -t, 0], [1, -t, 0], [0, -1, t], [0, 1, t], [0, -1, -t], [0, 1, -t],
         [t, 0, -1], [t, 0, 1], [-t, 0, -1], [-t, 0, 1]]
    f = [[0, 11, 5], [0, 5, 1], [0, 1, 7], [0, 7, 10], [0, 10, 11], [1, 5, 9], [5, 11, 4], [11, 10, 2], [10, 7, 6],
         [7, 1, 8], [3, 9, 4], [3, 4, 2], [3, 2, 6], [3, 6, 8], [3, 8, 9], [4, 9, 5], [2, 4, 11], [6, 2, 10],
         [8, 6, 7], [9, 8, 1]]
    v = np.array(v, np.float64)
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    f = np.array(f, np.int64)
    for _ in range(level):
        cache = {}
        verts = list(v)

        def mid(i, j):
            k = (min(i, j), max(i, j))
            if k not in cache:
                m = verts[i] + verts[j]
                verts.append(m / np.linalg.norm(m))
                cache[k] = len(verts) - 1
            return cache[k]

        nf = []
        for a, b, c in f:
            ab, bc, ca = mid(a, b), mid(b, c), mid(c, a)
            nf += [[a, ab, ca], [b, bc, ab], [c, ca, bc], [ab, bc, ca]]
        v, f = np.array(verts), np.array(nf, np.int64)
    return (v * radius).astype(np.float32), f.astype(np.int32)


def head(n_lat: int = 70, n_lon: int = 72, seed: int = 3):
    """A bumpy ellipsoid: a latitude-longitude grid of n_lat - 1 rings plus two poles."""
    rng = np.random.default_rng(seed)
    th = np.linspace(0, math.pi, n_lat + 1)[1:-1]
    ph = np.linspace(0, 2 * math.pi, n_lon, endpoint=False)
    T, Pp = np.meshgrid(th, ph, indexing="ij")
    amp = rng.normal(0, 0.02, (4,))
    bump = 1 + amp[0] * np.sin(3 * Pp) * np.sin(T) + amp[1] * np.cos(2 * T) + amp[2] * np.sin(5 * T + Pp) \
        + amp[3] * np.cos(4 * Pp)
    ax = np.array([0.078, 0.095, 0.088])
    ring = np.stack([np.sin(T) * np.cos(Pp), np.sin(T) * np.sin(Pp), np.cos(T)], -1) * ax * bump[..., None]
    v = np.concatenate([ring.reshape(-1, 3), [[0, 0, ax[2]], [0, 0, -ax[2]]]])
    R, L = n_lat - 1, n_lon
    top, bot = R * L, R * L + 1
    idx = lambda r, c: r * L + c % L  # noqa: E731
    f = []
    for c in range(L):
        f.append([top, idx(0, c), idx(0, c + 1)])
        f.append([bot, idx(R - 1, c + 1), idx(R - 1, c)])
        for r in range(R - 1):
            f.append([idx(r, c), idx(r + 1, c), idx(r + 1, c + 1)])
            f.append([idx(r, c), idx(r + 1, c + 1), idx(r, c + 1)])
    return v.astype(np.float32), np.array(f, np.int32)


def head_holes():
    v, f = head()
    cen = v[f].astype(np.float64).mean(1)
    d = cen / np.linalg.norm(cen, axis=1, keepdims=True)
    keep = np.ones(len(f), bool)
    for axis, cos in (([0.5, 0.75, 0.2], 0.985), ([-0.5, 0.75, 0.2], 0.985), ([0, 0.85, -0.5], 0.97),
                      ([0, 0, -1], 0.93), ([0.3, -0.2, 0.93], 0.995)):
        a = np.array(axis) / np.linalg.norm(axis)
        keep &= d @ a < cos
    return v, f[keep]


def degenerate():
    v, f = icosphere(2, 0.1)
    rng = np.random.default_rng(5)
    extra_v = np.array([[0.02, 0.0, 0.0], [0.05, 0.0, 0.0], [0.08, 0.0, 0.0],       # collinear along x (n = 0 exactly)
                        [0.0, 0.03, 0.03], [0.0, 0.06, 0.06],                        # a segment along (0, 1, 1)
                        [-0.04, -0.04, 0.01],                                        # a point
                        [0.01, 0.01, 0.01], [0.02, 0.02, 0.02], [0.04, 0.04, 0.04]], np.float32)
    V = len(v)
    v = np.concatenate([v, extra_v])
    extra_f = [[V, V + 1, V + 2], [V + 3, V + 4, V + 3], [V + 5, V + 5, V + 5], [V + 6, V + 8, V + 7],
               [V + 2, V, V + 1]]
    dup = f[rng.choice(len(f), 12, replace=False)]
    f = np.concatenate([f, np.array(extra_f, np.int32), dup])
    return v.astype(np.float32), f.astype(np.int32)


def big():
    return icosphere(6, 0.1)


MESHES = {"icosphere": lambda: icosphere(3), "head": head, "head_holes": head_holes, "degenerate": degenerate,
          "big": big}


def queries(verts: np.ndarray, faces: np.ndarray, n: int, seed: int) -> np.ndarray:
    """(M,3) float32: on the surface, near vertices and edges, inside and outside, far away, and six non-finite
    rows.  n sets the size of each group."""
    rng = np.random.default_rng(seed)
    v = verts.astype(np.float64)
    tri = v[faces[rng.integers(0, len(faces), n)]]
    bary = rng.dirichlet([1, 1, 1], n)
    surface = np.einsum("nk,nkj->nj", bary, tri)
    vert = v[rng.integers(0, len(v), n)] + rng.normal(0, 1, (n, 3)) * 10.0 ** rng.uniform(-7, -3, (n, 1))
    e = faces[rng.integers(0, len(faces), n)]
    t = rng.random((n, 1))
    edge = v[e[:, 0]] * t + v[e[:, 1]] * (1 - t) + rng.normal(0, 1, (n, 3)) * 10.0 ** rng.uniform(-7, -3, (n, 1))
    lo, hi = v.min(0), v.max(0)
    box = lo - 0.25 * (hi - lo) + rng.random((n, 3)) * 1.5 * (hi - lo)
    far = rng.normal(0, 1, (n // 4 + 1, 3))
    far *= (10.0 ** rng.uniform(0, 2, (len(far), 1))) / np.linalg.norm(far, axis=1, keepdims=True)
    bad = np.array([[np.nan, 0, 0], [0, np.inf, 0], [0, 0, -np.inf], [np.nan] * 3, [1e30, np.nan, 0], [0, 0, np.inf]])
    return np.concatenate([surface, vert, edge, box, far, bad]).astype(np.float32)


def gaussians(verts: np.ndarray, faces: np.ndarray, P: int, seed: int):
    """A Gaussian scene scattered across the surface: xyz on a random face, pushed along the normal by up to 1 cm;
    activated scaling exp(N(-6, 1)) (0.3 mm to 7 mm); raw unnormalised rotations; activated labels in (0, 1).
    -> xyz (P,3), scaling (P,3), rotation (P,4), label (P,1), float32."""
    rng = np.random.default_rng(seed)
    v = verts.astype(np.float64)
    tri = v[faces[rng.integers(0, len(faces), P)]]
    bary = rng.dirichlet([1, 1, 1], P)
    n = np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0])
    n /= np.linalg.norm(n, axis=1, keepdims=True)
    xyz = np.einsum("nk,nkj->nj", bary, tri) + n * rng.uniform(-0.01, 0.01, (P, 1))
    scaling = np.exp(rng.normal(-6, 1, (P, 3)))
    rotation = rng.normal(0, 1, (P, 4)) * rng.uniform(0.5, 2.0, (P, 1))
    label = 1 / (1 + np.exp(-rng.normal(0, 3, (P, 1))))
    return tuple(a.astype(np.float32) for a in (xyz, scaling, rotation, label))
