"""Kernel times and the idle gaps between them in the benchmark step, from a `torch.profiler` trace.

    python tools/step_gaps.py [--steps 24] [--out step_gaps.json]

Runs the workload of `bench.py` (oracle/synth.py strand scene, seed 0, 1920x1080, 8 views cycled, `_C` forward
followed by `rasterize_gaussians_backward_arena`) under `torch.profiler` with CUDA activities and writes one JSON
file: per position in the step, every device operation (kernel or memset) with its median duration and the median
idle time of the GPU before it, plus the card's name and power limit read in the same run.  The gap before the first
operation of a step is the host's time between two steps and is reported on its own (`step_boundary_us`).
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clock = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as exc:      # the figures stay usable without the card line; say why it is missing
        return {"error": str(exc)}


def device_ops(trace_path):
    """Kernels and memsets of a chrome trace in start order: [(name, start_us, dur_us)]."""
    with open(trace_path) as f:
        ev = json.load(f)["traceEvents"]
    ops = [(e["name"], float(e["ts"]), float(e["dur"])) for e in ev
           if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memset")]
    ops.sort(key=lambda o: o[1])
    return ops


def short(name):
    """A kernel's name without its namespace prefix and parameter list (template arguments kept)."""
    name = name.replace("(anonymous namespace)::", "")
    if name.startswith("void "):
        name = name[5:]
    depth = 0
    for i, ch in enumerate(name):
        if ch == "<":
            depth += 1
        elif ch == ">":
            depth -= 1
        elif ch == "(" and depth == 0:
            return name[:i]
    return name


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=24)
    ap.add_argument("--warmup", type=int, default=8)
    ap.add_argument("--out", default="step_gaps.json")
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    from gaussianhaircut_b200 import _C
    import synth

    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    W, H = 1920, 1080
    scene = synth.make_strand_scene(5000, seed=0)
    views = [synth.rasterizer_inputs(scene, synth.make_camera((v * 8) % 64, W, H), mode="native", device=dev) for v in range(8)]
    dL = synth.upstream_gradient(W, H, 0).to(dev)
    e = torch.Tensor([])

    def step(i):
        kw, s = views[i % 8]["kwargs"], views[i % 8]["settings"]
        g = lambda k: e if kw[k] is None else kw[k]  # noqa: E731
        R, color, radii, geom, binning, img = _C.rasterize_gaussians(
            s["bg"], kw["means3D"], kw["means2D"], g("colors_precomp"), kw["opacities"], g("scales"), g("rotations"),
            s["scale_modifier"], g("cov3D_precomp"), g("conic_precomp"), s["viewmatrix"], s["projmatrix"], s["tanfovx"],
            s["tanfovy"], H, W, e, s["sh_degree"], s["campos"], s["prefiltered"], False)
        _C.rasterize_gaussians_backward_arena(
            s["bg"], kw["means3D"], radii, g("colors_precomp"), g("scales"), g("rotations"), s["scale_modifier"],
            g("cov3D_precomp"), g("conic_precomp"), s["viewmatrix"], s["projmatrix"], s["tanfovx"], s["tanfovy"], dL, e,
            s["sh_degree"], s["campos"], geom, R, binning, img, False)

    for i in range(args.warmup):
        step(i)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for i in range(args.steps):
            step(i)
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "trace.json")
        prof.export_chrome_trace(path)
        ops = device_ops(path)

    # a step starts with the memset of the tile histogram that precedes the preprocess kernel
    starts = [i for i, (n, _, _) in enumerate(ops) if short(n).startswith("gh_preprocess_kernel")]
    starts = [i - 1 if i > 0 and ops[i - 1][0].startswith("Memset") else i for i in starts]
    if not starts:
        raise SystemExit(f"no gh_preprocess_kernel among the {len(ops)} device operations of the trace")
    steps = [ops[a:b] for a, b in zip(starts, starts[1:] + [len(ops)])]
    shape = [short(n) for n, _, _ in steps[0]]
    same = [s for s in steps if [short(n) for n, _, _ in s] == shape]
    table, boundary = [], []
    for k, name in enumerate(shape):
        durs = [s[k][2] for s in same]
        gaps = [s[k][1] - (s[k - 1][1] + s[k - 1][2]) for s in same] if k > 0 else []
        table.append({"op": name, "dur_us": round(statistics.median(durs), 2),
                      "gap_before_us": round(statistics.median(gaps), 2) if gaps else None})
    for a, b in zip(steps, steps[1:]):
        boundary.append(b[0][1] - (a[-1][1] + a[-1][2]))
    inner_gaps = sum(r["gap_before_us"] for r in table[1:])
    memset_us = sum(r["dur_us"] for r in table if r["op"].startswith("Memset"))
    span = [s[-1][1] + s[-1][2] - s[0][1] for s in same]
    result = {
        "card": card(),
        "workload": "bench.py --gpus 1: 5000 strands (500 k Gaussians), 1920x1080, 8 views, native mode",
        "steps_traced": len(steps), "steps_used": len(same),
        "ops": table,
        "sum_op_us": round(sum(r["dur_us"] for r in table), 2),
        "sum_gaps_in_step_us": round(inner_gaps, 2),
        "memset_us": round(memset_us, 2),
        "step_span_us": round(statistics.median(span), 2),
        "step_boundary_us": round(statistics.median(boundary), 2) if boundary else None,
    }
    with open(args.out, "w") as f:
        json.dump(result, f, indent=1)
    w = max(len(r["op"]) for r in table)
    for r in table:
        gap = "" if r["gap_before_us"] is None else f"{r['gap_before_us']:8.2f}"
        print(f"{r['op']:<{w}}  {r['dur_us']:8.2f}  {gap}")
    print(json.dumps({k: v for k, v in result.items() if k != "ops"}))


if __name__ == "__main__":
    main()
