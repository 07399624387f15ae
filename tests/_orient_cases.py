"""Seeded test images for the orientation-map tests (tests/test_gpu_orient.py, tools/orient_*.py)."""
from __future__ import annotations

import math
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if os.path.join(ROOT, "oracle") not in sys.path:
    sys.path.insert(0, os.path.join(ROOT, "oracle"))

# TOL of oracle/orient64.check: a kernel variance may lie TOL * var_scale from the float64 replay's.  var_scale is the
# first-order float32 error bound over u = 2^-24, so TOL = u is that bound itself; tools/orient_replay_calibrate.py
# measures how much of it the kernels use (DESIGN §15).
TOL = 2.0 ** -24
# The reference's cuDNN convolution is held to the replay with TF32 input rounding (oracle/orient64.replay(tf32=True)):
# its variances to the matching multiple of the same scale, (2^-9 + 2^-20) / (17 * 17) + TOL.
TOL_REF = (2.0 ** -9 + 2.0 ** -20) / 289 + TOL


def noise(H: int, W: int, seed: int, C: int = 3) -> np.ndarray:
    return np.random.default_rng(seed).integers(0, 256, (H, W, C), dtype=np.uint8)


def strands(H: int, W: int, seed: int, C: int = 3, n: int = 1500) -> np.ndarray:
    """A hair-like picture: n anti-aliased random-walk polylines of 1-2 px width in brown-to-blond tones on a dark
    background with a soft face-coloured blob, quantised to uint8 (RGBA: alpha is a ramp, which the maps ignore)."""
    import cv2
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:H, 0:W]
    img = np.zeros((H, W, 3), np.float64)
    blob = np.exp(-(((x - W * 0.5) / (W * 0.18)) ** 2 + ((y - H * 0.6) / (H * 0.25)) ** 2))
    img += blob[..., None] * np.array([120.0, 150.0, 200.0])
    img = img.astype(np.uint8)
    for _ in range(n):
        p = np.array([rng.uniform(0.2, 0.8) * W, rng.uniform(0.05, 0.5) * H])
        a = rng.uniform(0, 2 * math.pi)
        pts = [p.copy()]
        for _ in range(int(rng.integers(20, 60))):
            a += rng.normal(0, 0.12)
            p = p + 6.0 * np.array([math.cos(a), abs(math.sin(a)) + 0.3])
            pts.append(p.copy())
        tone = rng.uniform(0.2, 1.0)
        colour = (int(40 + 80 * tone), int(60 + 120 * tone), int(90 + 150 * tone))
        cv2.polylines(img, [np.round(np.array(pts) * 16).astype(np.int32)], False, colour, int(rng.integers(1, 3)),
                      cv2.LINE_AA, shift=4)
    if C == 4:
        alpha = (np.linspace(0, 255, W)[None, :] * np.ones((H, 1))).astype(np.uint8)
        img = np.concatenate([img, alpha[..., None]], axis=2)
    return np.ascontiguousarray(img)


def grating(deg: float, size: int = 128, f: float = 0.23) -> np.ndarray:
    """A sinusoidal grating whose stripes run at `deg` degrees, uint8 RGB."""
    phi = math.radians(deg)
    y, x = np.mgrid[0:size, 0:size]
    g = np.round(128 + 100 * np.cos(2 * math.pi * f * (x * math.cos(phi) + y * math.sin(phi)))).astype(np.uint8)
    return np.ascontiguousarray(np.repeat(g[..., None], 3, axis=2))


def crops(H: int, W: int, size: int, seed: int, n: int):
    """The four corners and n seeded interior crops (y0, y1, x0, x1) of at most size x size pixels."""
    rng = np.random.default_rng(seed)
    s_y, s_x = min(size, H), min(size, W)
    out = [(0, s_y, 0, s_x), (0, s_y, W - s_x, W), (H - s_y, H, 0, s_x), (H - s_y, H, W - s_x, W)]
    for _ in range(n):
        y0, x0 = int(rng.integers(0, H - s_y + 1)), int(rng.integers(0, W - s_x + 1))
        out.append((y0, y0 + s_y, x0, x0 + s_x))
    return out
