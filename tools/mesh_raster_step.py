"""Time the mesh rasterizer at the scalp script's scale and print one JSON line (DESIGN §24).

    python tools/mesh_raster_step.py [--views 128] [--reps 5]

For the ~10 k- and ~40 k-face heads of tests/_sdf_cases.py, 128 views on a sphere of cameras, at 1024 x 1024 and
2048 x 2048: `rasterize_faces` and `scalp_visibility` end to end (CUDA events around each call after a warm-up,
median, min and max), pixels per second and (face, pixel-in-box) pairs per second -- the pairs the raster kernel
walks, counted by the host harness's copy of the setup arithmetic -- and the card's name and power limit, read in the
same run.  There is no pytorch3d arm: pytorch3d is not part of this package's environment.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import _meshraster64 as O  # noqa: E402
import _sdf_cases as K  # noqa: E402
from gaussianhaircut_b200 import mesh as M  # noqa: E402


def box_pairs(v, f, Ks, Rs, ts, H, W) -> int:
    """Sum over views and faces of the pixel boxes the raster kernel walks (the setup arithmetic on the host)."""
    import tempfile
    src = os.path.join(ROOT, "tests", "host_harness", "mesh_raster_host.cpp")
    so = os.path.join(tempfile.mkdtemp(prefix="gh_mr_"), "libmr.so")
    subprocess.run(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-std=c++17", "-w", src, "-o", so],
                   check=True)
    h = C.CDLL(so)
    ptr = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    F = len(f)
    rec = np.zeros((F, 20), np.float32)
    code = np.empty(F, np.int32)
    total = 0
    for b in range(len(Ks)):
        h.gh_host_raster_setup(len(v), F, ptr(v), ptr(f), ptr(np.ascontiguousarray(Ks[b])),
                               ptr(np.ascontiguousarray(Rs[b])), ptr(np.ascontiguousarray(ts[b])), H, W, ptr(rec),
                               ptr(code))
        nj, ni = rec[:, 18].view(np.int32).astype(np.int64), rec[:, 19].view(np.int32).astype(np.int64)
        total += int((nj * ni).sum())
    return total


def _times(fn, reps):
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return {"median_ms": round(float(np.median(ts)), 3), "min_ms": round(float(np.min(ts)), 3),
            "max_ms": round(float(np.max(ts)), 3)}


def measure(label, v, f, B, H, W, reps, dev):
    Ks, Rs, ts = O.sphere_cameras(B, H, W, 49, radius=0.45, f_scale=1.6)
    dv = [torch.from_numpy(np.ascontiguousarray(x)).to(dev) for x in (v, f, Ks, Rs, ts)]
    rows = torch.arange(H, device=dev)[:, None]
    cut = torch.from_numpy(np.random.default_rng(5).uniform(0.3, 0.7, B)).to(dev)
    head = (rows[None] >= (cut * H)[:, None, None]).expand(B, H, W).contiguous()
    for _ in range(2):
        M.rasterize_faces(*dv, H, W)
        M.scalp_visibility(*dv, head, chunk=16)
    torch.cuda.synchronize()
    r = _times(lambda: M.rasterize_faces(*dv, H, W), reps)
    s = _times(lambda: M.scalp_visibility(*dv, head, chunk=16), reps)
    pairs = box_pairs(v, f, Ks, Rs, ts, H, W)
    px = B * H * W
    return {"mesh": label, "faces": int(len(f)), "views": B, "H": H, "W": W, "rasterize_faces": r,
            "scalp_visibility": s, "box_pairs": pairs,
            "rasterize_pixels_per_s": px / (r["median_ms"] * 1e-3), "rasterize_pairs_per_s": pairs / (r["median_ms"] * 1e-3),
            "scalp_pixels_per_s": px / (s["median_ms"] * 1e-3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=128)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mesh_raster_step: needs a CUDA device")
    dev = torch.device("cuda:0")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    rows = []
    for label, (v, f) in (("head ~10 k faces", K.head()), ("head ~40 k faces", K.head(140, 144))):
        for side in (1024, 2048):
            rows.append(measure(label, v, f, args.views, side, side, args.reps, dev))
    print(json.dumps({"card": smi[0] if smi else torch.cuda.get_device_name(dev), "rows": rows}))


if __name__ == "__main__":
    main()
