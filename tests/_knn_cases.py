"""Seeded point clouds of the distCUDA2 tests and of tools/knn_case.py (test infrastructure), and the numpy float32
restatement of the contract they are checked with."""
from __future__ import annotations

import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if os.path.join(ROOT, "oracle") not in sys.path:
    sys.path.insert(0, os.path.join(ROOT, "oracle"))


def uniform(P: int, seed: int = 0) -> np.ndarray:
    """(a) uniform in the unit cube."""
    return np.random.default_rng(seed).random((P, 3), dtype=np.float32)


def head_shell(P: int, seed: int = 0) -> np.ndarray:
    """(b) what a COLMAP cloud of a head looks like: a shell of radius 0.1 with 1e-3 noise, plus 1 % outliers in a box
    100x larger than the head's."""
    rng = np.random.default_rng(seed)
    n_out = P // 100
    d = rng.standard_normal((P - n_out, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    shell = d * 0.1 + 1e-3 * rng.standard_normal((P - n_out, 3))
    out = rng.uniform(-10.0, 10.0, (n_out, 3))
    pts = np.concatenate([shell, out]).astype(np.float32)
    return pts[rng.permutation(P)]


def strand_vertices(P: int, seed: int = 0) -> np.ndarray:
    """(c) segment midpoints of `synth.make_strand_scene` strands (100 per strand, 2e-3 apart): anisotropic, with
    near-duplicates along the strands.  Built 1000 strands at a time."""
    import synth
    parts, left, k = [], P, 0
    while left > 0:
        n = min(1000, (left + 99) // 100)
        parts.append(synth.make_strand_scene(n, seed=seed * 100003 + k)["xyz"].numpy()[:left])
        left -= parts[-1].shape[0]
        k += 1
    return np.concatenate(parts) if parts else np.zeros((0, 3), np.float32)


def lattice(n: int = 64, seed: int = 0) -> np.ndarray:
    """(d) an n^3 integer lattice in random order: every point has six neighbours at exactly 1."""
    g = np.stack(np.meshgrid(*(np.arange(n, dtype=np.float32),) * 3, indexing="ij"), -1).reshape(-1, 3)
    return g[np.random.default_rng(seed).permutation(g.shape[0])]


def repeated(P: int, seed: int = 0) -> np.ndarray:
    """(e) about P points: each of P // 2.5 uniform points repeated 1-4 times, in random order."""
    rng = np.random.default_rng(seed)
    base = rng.random((max(1, int(P / 2.5)), 3), dtype=np.float32)
    pts = np.repeat(base, rng.integers(1, 5, base.shape[0]), axis=0)
    return pts[rng.permutation(pts.shape[0])]


def one_point(P: int = 10000, seed: int = 0) -> np.ndarray:
    """(f) P copies of one point: every result is 0."""
    return np.tile(np.array([[0.3, -0.2, 0.7]], np.float32), (P, 1))


def offset_cube(P: int, seed: int = 0) -> np.ndarray:
    """(g) a cube of extent 1e-2 centred at (1e4, -1e4, 1e4): dx cancels most of the coordinates' bits."""
    rng = np.random.default_rng(seed)
    return (np.array([1e4, -1e4, 1e4]) + (rng.random((P, 3)) - 0.5) * 1e-2).astype(np.float32)


def nonfinite(P: int, seed: int = 0) -> np.ndarray:
    """(i) uniform points, about 5 % of the rows with a NaN, +inf or -inf in one or more coordinates."""
    rng = np.random.default_rng(seed)
    pts = rng.random((P, 3), dtype=np.float32)
    bad = rng.random(P) < 0.05
    vals = np.array([np.nan, np.inf, -np.inf], np.float32)
    for k in range(3):
        hit = bad & (rng.random(P) < 0.5)
        pts[hit, k] = vals[rng.integers(0, 3, int(hit.sum()))]
    pts[bad & np.isfinite(pts).all(1), 0] = np.nan
    return pts


def tiny(P: int, seed: int = 0) -> np.ndarray:
    """(h) P = 0 ... 5."""
    return uniform(P, seed)


# name -> (generator, size of the bit-exact CPU comparison (P <= 3000), size of the GPU comparison)
CASES = {
    "a_uniform": (uniform, 3000, 200_000),
    "b_head_shell": (head_shell, 3000, 200_000),
    "c_strands": (strand_vertices, 3000, 100_000),
    "d_lattice": (lambda P, seed=0: lattice(round(P ** (1 / 3)), seed), 14 ** 3, 64 ** 3),
    "e_repeated": (repeated, 3000, 100_000),
    "f_one_point": (one_point, 3000, 10_000),
    "g_offset_cube": (offset_cube, 3000, 100_000),
    "i_nonfinite": (nonfinite, 3000, 100_000),
}


def brute_mean_dist3(pts) -> np.ndarray:
    """The contract restated with numpy float32 arithmetic over all pairs (every operation rounded on its own)."""
    pts = np.ascontiguousarray(np.asarray(pts, np.float32).reshape(-1, 3))
    P = pts.shape[0]
    out = np.full(P, np.nan, np.float32)
    fin = np.isfinite(pts).all(axis=1)
    q, idx = pts[fin], np.nonzero(fin)[0]
    n = q.shape[0]
    for a in range(0, n, 256):
        p = q[a:a + 256]
        dx = q[None, :, 0] - p[:, None, 0]
        dy = q[None, :, 1] - p[:, None, 1]
        dz = q[None, :, 2] - p[:, None, 2]
        s = np.concatenate([(dx * dx + dy * dy) + dz * dz, np.full((p.shape[0], 3), np.inf, np.float32)], axis=1)
        s[np.arange(p.shape[0]), np.arange(a, a + p.shape[0])] = np.inf        # j != i by index, not by position
        b = np.sort(np.partition(s, 2, axis=1)[:, :3], axis=1)
        out[idx[a:a + p.shape[0]]] = ((b[:, 0] + b[:, 1]) + b[:, 2]) / np.float32(3.0)
    return out


def assert_same_bits(got, want, what: str = ""):
    """Bit-identical float32 arrays, NaN matching NaN."""
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    assert got.shape == want.shape, f"{what}: shape {got.shape} vs {want.shape}"
    gn, wn = np.isnan(got), np.isnan(want)
    assert np.array_equal(gn, wn), f"{what}: NaN at {np.nonzero(gn != wn)[0][:8]}"
    diff = np.nonzero(got[~gn].view(np.uint32) != want[~wn].view(np.uint32))[0]
    assert diff.size == 0, (f"{what}: {diff.size} of {got.size} differ, e.g. {got[~gn][diff[:4]]} vs "
                            f"{want[~wn][diff[:4]]}")
