"""Per-view cost of the render scripts' sweep and of training_report, eager PyTorch composition against the inference
module, on the current GPU:  python tools/render_set_step.py [--views 12] [--repeats 5] [--small]

  (a) renderer.render / render_hair_strands under no_grad + the reference's epilogue, vis_orient, masking and
      save_image quantisation in PyTorch + .cpu() per saved map (what src/render_gaussians.py:50-68 does per view)
  (b) ViewRenderer.render_maps + sweep into pinned host buffers
and the training_report loop body in PyTorch against evaluate_views.  Shapes: the stage-1 model (500 k Gaussians) and
the strand model (30 000 x 99 segments + 200 k head blobs) at 1920x1080 and 960x540, synthetic scenes of oracle/synth.py.
Device time is the CUDA-event time around the whole sweep, host time the wall clock around it ending in a
synchronise; both per view, median of the repeats after one warm-up sweep.  PNG encoding is CPU work that both arms
share; it is timed on its own for one view.  Nothing about clocks or power is set: the card's name and power limit are
printed with the numbers."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")]
import synth  # noqa: E402
import ref_python  # noqa: E402
import _strands  # noqa: E402
from test_gpu_render_maps import _gaussians, _head, _strand_model, _training_report, _vis_orient  # noqa: E402

PIPE = types.SimpleNamespace(debug=False)


def _views(dev, n, W, H):
    g = torch.Generator().manual_seed(1)
    out = []
    for k in range(n):
        v = ref_python.make_camera(synth.make_camera((5 * k) % 64, W, H), dev)
        v.image_name = f"v{k}.png"
        v.original_image, v.original_orient_angle = torch.rand(3, H, W, generator=g), torch.rand(1, H, W, generator=g)
        v.original_mask, v.original_orient_conf = (torch.rand(2, H, W, generator=g) > 0.3).float(), torch.rand(1, H, W, generator=g)
        out.append(v)
    return out


def _eager_view(render, view):
    """render_set's loop body with the file writes replaced by the device -> host copies save_image / torch.save make."""
    o = render(view)
    hair = o["mask"][:1]
    conf = o["orient_conf"] * hair
    maps = (o["render"], hair, o["mask"][1:], o["orient_angle"] * hair, _vis_orient(o["orient_angle"], hair),
            _vis_orient(o["orient_angle"], 1 - 1 / (conf + 1)))
    host = [m.mul(255).add_(0.5).clamp_(0, 255).permute(1, 2, 0).to("cpu", torch.uint8) for m in maps]
    host.append(conf.cpu())
    return host


def _timed(fn, repeats):
    dev_ms, wall_ms = [], []
    for r in range(repeats + 1):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        e0.record()
        n = fn()
        e1.record()
        torch.cuda.synchronize()
        if r:
            wall_ms.append((time.perf_counter() - t0) * 1e3 / n)
            dev_ms.append(e0.elapsed_time(e1) / n)
    return {"device_ms_per_view": round(statistics.median(dev_ms), 3), "wall_ms_per_view": round(statistics.median(wall_ms), 3),
            "wall_ms_min_max": [round(min(wall_ms), 3), round(max(wall_ms), 3)]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=12)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--small", action="store_true", help="tiny models (a rehearsal of the script, not a measurement)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("render_set_step: needs a GPU (a CPU run measures nothing)")
    from gaussianhaircut_b200 import inference, renderer
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": q, "views": a.views, "repeats": a.repeats, "method": __doc__.split("Device time")[1][:180]}))
    bg = torch.tensor(synth.BG_DEFAULT, device=dev)
    shapes = {"stage1": (2000 if a.small else 500000, None), "strands": (200 if a.small else 30000, 2000 if a.small else 200000)}
    for shape, (n, n_head) in shapes.items():
        if n_head is None:
            pc = _gaussians(dev, n)
            args, kw = (pc, PIPE, bg), {}
            render = lambda v: renderer.render(v, pc, PIPE, bg)  # noqa: E731
            stage = "appearance"
        else:
            head, hair = _head(dev, n_head), _strand_model(dev, n, 99)
            args, kw = (head, PIPE, bg), {"pc_hair": hair}
            render = lambda v: renderer.render_hair_strands(v, head, hair, PIPE, bg)  # noqa: E731
            stage = "strands"
        for W, H in ((1920, 1080), (960, 540)):
            views = _views(dev, a.views, W, H)
            vr = inference.ViewRenderer(*args, **kw)
            want = tuple(inference.RENDER_SET_MAPS.values())

            def eager():
                with torch.no_grad():
                    for v in views:
                        _eager_view(render, v)
                return len(views)

            def fused():
                for _v, _m in inference.sweep(vr, views, want):
                    pass
                return len(views)

            def raw_only():
                for v in views:
                    vr.render_raw(v, check=False)
                return len(views)

            def maps_only():
                raw = vr._bufs["raw"]
                for _ in views:
                    vr.maps_of(raw, want)
                return len(views)

            def report_eager():
                with torch.no_grad():
                    _training_report(views, render, stage)
                return len(views)

            def report_fused():
                inference.evaluate_views(views, vr, stage)
                return len(views)

            res = {"shape": shape, "W": W, "H": H}
            for name, fn in (("sweep_pytorch", eager), ("sweep_inference", fused), ("render_raw_only", raw_only),
                             ("gh_render_maps_only", maps_only), ("report_pytorch", report_eager), ("report_inference", report_fused)):
                res[name] = _timed(fn, a.repeats)
            res["retries"], res["allocations"] = vr.retries, vr.allocations
            v, m = next(iter(inference.sweep(vr, views[:2], want)))
            m = {k: t.clone() for k, t in m.items()}
            t0 = time.perf_counter()
            with tempfile.TemporaryDirectory() as tmp:
                for d, k in inference.RENDER_SET_MAPS.items():
                    if k != "orient_conf_masked":
                        inference.save_png(m[k], os.path.join(tmp, d + ".png"))
            res["png_encode_wall_ms_per_view"] = round((time.perf_counter() - t0) * 1e3, 1)
            print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
