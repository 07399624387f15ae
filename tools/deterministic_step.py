"""What the deterministic blend backward costs: the bench.py workload (native call shape, 1920x1080, strands(5000) =
500 000 Gaussians, 8 views, forward + arena backward) with the default and the deterministic path alternating in one
process (torch.use_deterministic_algorithms off / on), 5 repeats of a K-step window each.

    python tools/deterministic_step.py [--steps 30] [--repeats 5] [--out DIR]

Prints one JSON line: the card and its power limit; per path the median ms per step, the blend_backward stage time
(gh_stage_timing), and -- from a torch.profiler run of its own -- the split of the deterministic stage into the offset
scan, the per-tile walk and the gather; and the largest norm-relative difference between the two paths' gradients."""
import argparse, json, os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "oracle"))
ap = argparse.ArgumentParser()
ap.add_argument("--strands", type=int, default=5000)
ap.add_argument("--steps", type=int, default=30)
ap.add_argument("--repeats", type=int, default=5)
ap.add_argument("--out", default=None, help="directory for the profiler trace")
args = ap.parse_args()
import torch
from gaussianhaircut_b200 import _C, _capi
import synth

dev = torch.device("cuda:0")
W, H = 1920, 1080
scene = synth.make_strand_scene(args.strands, seed=0)
views = [synth.rasterizer_inputs(scene, synth.make_camera((v * 8) % 64, W, H), mode="native", device=dev) for v in range(8)]
dL = synth.upstream_gradient(W, H, 0).to(dev)
e = torch.Tensor([])


def step(i):
    inp = views[i % 8]; kw, s = inp["kwargs"], inp["settings"]
    g = lambda k: e if kw[k] is None else kw[k]  # noqa: E731
    R, color, radii, geom, binning, img = _C.rasterize_gaussians(
        s["bg"], kw["means3D"], kw["means2D"], g("colors_precomp"), kw["opacities"], g("scales"), g("rotations"), 1.0,
        g("cov3D_precomp"), g("conic_precomp"), s["viewmatrix"], s["projmatrix"], s["tanfovx"], s["tanfovy"], H, W, e, 3,
        s["campos"], s["prefiltered"], False)
    flat, _g, _sh = _C.rasterize_gaussians_backward_arena(
        s["bg"], kw["means3D"], radii, g("colors_precomp"), g("scales"), g("rotations"), 1.0, g("cov3D_precomp"),
        g("conic_precomp"), s["viewmatrix"], s["projmatrix"], s["tanfovx"], s["tanfovy"], dL, e, 3, s["campos"], geom, R,
        binning, img, False)
    return flat


def window(det):
    torch.use_deterministic_algorithms(det)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(args.steps):
        step(i)
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / args.steps


def stage_us(det):
    torch.use_deterministic_algorithms(det)
    lib = _capi.load()
    lib.gh_stage_timing_enable(1)
    for i in range(16):
        step(i)
    torch.cuda.synchronize()
    st = _capi.stage_timing_read()
    lib.gh_stage_timing_enable(0)
    ms, c = st["blend_backward"]
    return 1e3 * ms / c


for det in (False, True):                                   # warm-up of both paths
    torch.use_deterministic_algorithms(det)
    for i in range(8):
        step(i)
torch.cuda.synchronize()
times = {"default": [], "deterministic": []}
for r in range(args.repeats):
    for name, det in (("default", False), ("deterministic", True)):
        times[name].append(window(det))
med = lambda v: sorted(v)[len(v) // 2]  # noqa: E731
res = {name: {"ms_per_step_median": round(med(v), 4), "ms_per_step_all": [round(x, 4) for x in v]} for name, v in times.items()}
for name, det in (("default", False), ("deterministic", True)):
    res[name]["blend_backward_us"] = round(stage_us(det), 1)

# kernel split of the deterministic stage: torch.profiler, a run of its own
from torch.profiler import profile, ProfilerActivity
torch.use_deterministic_algorithms(True)
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for i in range(8):
        step(i)
    torch.cuda.synchronize()
split = {"scan": 0.0, "walk": 0.0, "gather": 0.0}
for ev in prof.key_averages():
    n = ev.key
    t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
    if "gh_det_area_sums_kernel" in n or "gh_det_part_scan_kernel" in n or "gh_det_offsets_kernel" in n:
        split["scan"] += t
    elif "gh_blend_backward_kernel" in n and ("<true>" in n or "ILb1E" in n):
        split["walk"] += t
    elif "gh_det_gather_kernel" in n:
        split["gather"] += t
res["deterministic"]["split_us"] = {k: round(v / 8, 1) for k, v in split.items()}
if args.out:
    os.makedirs(args.out, exist_ok=True)
    prof.export_chrome_trace(os.path.join(args.out, "deterministic_step_trace.json"))

# gradients of the two paths on every view
worst = 0.0
for i in range(8):
    torch.use_deterministic_algorithms(False)
    a = step(i).clone()
    torch.use_deterministic_algorithms(True)
    b = step(i).clone()
    worst = max(worst, float((a - b).norm() / a.norm().clamp_min(1e-30)))
torch.use_deterministic_algorithms(False)
try:
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=30).stdout.strip()
except Exception:
    q = torch.cuda.get_device_name(0) + ", power limit not available"
res["gpu"] = q
res["max_norm_rel_diff_det_vs_default"] = worst
res["ratio_blend_backward"] = round(res["deterministic"]["blend_backward_us"] / res["default"]["blend_backward_us"], 2)
print(json.dumps(res), flush=True)
