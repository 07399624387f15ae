"""Forward + backward time of one strand-stage render (train_strands.py's shape) in three arms, one JSON line:

  fused           renderer.render_hair_strands: midpoints, strand geometry and projection in this repository's kernels
  torch-geometry  the reference's GaussianModelCurves.initialize_gaussians_hair() (PyTorch) + renderer.render_hair
  reference       initialize_gaussians_hair() + the reference's own render_hair on its own rasterizer (oracle/_ref)

Every arm renders the same synthetic model (tests/_strands.py polylines + a frozen head block of blobs) from the same
camera and back-propagates the same fixed random weights of the four maps into .grad of _dirs, the features,
_orient_conf and viewspace_points.  Per step: CUDA events around forward + backward; a repeat = `--steps` steps after
`--warmup`; the median of `--repeats` repeats is reported, with the card name and power limit read in the same call.
The `fused` maps are compared with the `torch-geometry` maps at the timed size: `maps_match` says whether every
norm-relative error is <= 1e-4 (1e-3 for orient_angle); the errors themselves are reported.

    python tools/strands_step.py [--strands 30000] [--segments 99] [--head 200000] [--width 1920 --height 1080]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def _card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        power = q.split(",")[-1].strip() if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--strands", type=int, default=30000)
    ap.add_argument("--segments", type=int, default=99)
    ap.add_argument("--head", type=int, default=200000)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--arms", default="fused,torch-geometry,reference")
    a = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("strands_step: no CUDA device (this measures the GPU; there is no CPU mode)")
    import _strands
    import ref_python
    import synth
    from gaussianhaircut_b200 import renderer

    dev = torch.device("cuda:0")
    W, H = a.width, a.height
    head = synth.make_blob_scene(a.head, seed=2, spread=0.08, max_scale=0.004) if a.head else _strands.empty_head_scene()
    poly = _strands.make_strand_polylines(a.strands, a.segments, seed=4)
    cam_d = synth.make_camera(7, W, H)
    bg = torch.tensor(synth.BG_DEFAULT, device=dev)
    g = torch.Generator().manual_seed(9)
    Wt = {k: torch.rand(c, H, W, generator=g).to(dev) for k, c in (("render", 3), ("mask", 2), ("orient_angle", 1), ("orient_conf", 1))}
    pipe = ref_python.pipe()
    arms = [s for s in a.arms.split(",") if s]

    def make_step(arm):
        pc, hair = _strands.make_curves_models(head, poly, dev)
        cam = ref_python.make_camera(cam_d, dev)
        if arm == "fused":
            fn = lambda: renderer.render_hair_strands(cam, pc, hair, pipe, bg)  # noqa: E731
        else:
            rh = renderer.render_hair if arm == "torch-geometry" else ref_python.load_renderer("ref").render_hair

            def fn():
                hair.initialize_gaussians_hair()
                return rh(cam, pc, hair, pipe, bg)

        def step():
            for n in _strands.CURVES_PARAMS:
                getattr(hair, n).grad = None
            pkg = fn()
            sum((pkg[k] * Wt[k]).sum() for k in Wt).backward()
            return pkg
        return step

    name, power = _card()
    res = {"tool": "strands_step", "strands": a.strands, "segments": a.segments, "P_hair": a.strands * a.segments,
           "head": a.head, "width": W, "height": H, "steps": a.steps, "warmup": a.warmup, "repeats": a.repeats,
           "card": name, "power_limit": power, "ms_per_step": {}, "repeats_ms": {}}
    maps = {}
    for arm in arms:
        step = make_step(arm)
        for _ in range(a.warmup):
            step()
        torch.cuda.synchronize()
        reps = []
        for _ in range(a.repeats):
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for _ in range(a.steps):
                step()
            t1.record()
            torch.cuda.synchronize()
            reps.append(t0.elapsed_time(t1) / a.steps)
        res["ms_per_step"][arm] = round(statistics.median(reps), 4)
        res["repeats_ms"][arm] = [round(r, 4) for r in reps]
        pkg = step()
        maps[arm] = {k: pkg[k].detach().clone() for k in Wt}
        del pkg
        del step
        torch.cuda.empty_cache()
    if "fused" in maps and "torch-geometry" in maps:
        err = {}
        for k in Wt:
            x, y = maps["fused"][k].double(), maps["torch-geometry"][k].double()
            err[k] = float((x - y).norm() / y.norm().clamp_min(1e-300))
        res["fused_vs_torch_geometry_rel_err"] = err
        res["maps_match"] = all(e <= (1e-3 if k == "orient_angle" else 1e-4) for k, e in err.items())
    print(json.dumps(res))


if __name__ == "__main__":
    main()
