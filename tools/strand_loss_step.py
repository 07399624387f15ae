"""Time the strand stages' image loss, one JSON line:

  loss_ms        the loss alone, forward + backward at --width x --height, per strand stage:
                   kernels    losses.strand_image_loss / latent_strand_image_loss on a (10,H,W) render
                   reference  the reference's own loss_utils (l1_loss, ssim, or_loss) composed as
                              train_strands.py:128-147 / train_latent_strands.py:130-152 compose them, autograd,
                              PyTorch's default (TF32) convolution settings
  iteration_ms   the train_strands.py iteration on the tools/strands_step.py scene (30 000 x 99 strands, 200 000 head
                 blobs, 1080p):
                   reference  render_hair_strands, the PyTorch loss, torch.optim.Adam after the three
                              `.grad.isnan().any()` host checks
                   kernels    render_hair_strands, strand_image_loss, FusedAdam with the device NaN flag

The arms alternate repeat by repeat; each repeat times `--steps` steps after `--warmup` untimed ones with CUDA events;
the median of `--repeats` repeats is reported with the card name and power limit read in the same call.

    python tools/strand_loss_step.py [--strands 30000] [--segments 99] [--head 200000] [--width 1920 --height 1080]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

LAMBDAS = {1: (0.8, 0.2, 0.2, 0.1), 2: (0.8, 0.0, 0.2, 0.1)}
LRS = {"_dirs": 1.6e-4, "_features_dc": 2.5e-3, "_features_rest": 2.5e-3 / 20.0, "_orient_conf": 0.05}


def _time(steps_by_arm, steps, warmup, repeats):
    """{arm: (median ms per step, [repeat ms])}, arms alternating repeat by repeat."""
    import torch
    for fn in steps_by_arm.values():
        for _ in range(warmup):
            fn()
    torch.cuda.synchronize()
    reps = {arm: [] for arm in steps_by_arm}
    for _ in range(repeats):
        for arm, fn in steps_by_arm.items():
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for _ in range(steps):
                fn()
            t1.record()
            torch.cuda.synchronize()
            reps[arm].append(t0.elapsed_time(t1) / steps)
    return {arm: (round(statistics.median(r), 4), [round(x, 4) for x in r]) for arm, r in reps.items()}


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
    a = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("strand_loss_step: no CUDA device (this measures the GPU; there is no CPU mode)")
    import _strand_loss64 as sl
    import _strands
    import ref_python
    import synth
    from strands_step import _card
    from gaussianhaircut_b200 import losses, renderer
    from gaussianhaircut_b200.optim import FusedAdam
    ref_python.load_renderer("ref")                       # the reference's sources on sys.path
    from utils import loss_utils as ref
    fns = (ref.l1_loss, ref.ssim, ref.or_loss)

    dev = torch.device("cuda:0")
    W, H = a.width, a.height
    g = torch.Generator().manual_seed(3)
    r = lambda *s: torch.rand(*s, generator=g).to(dev)   # noqa: E731
    render = torch.cat([r(5, H, W), r(3, H, W) * 2 - 1, r(1, H, W) * 0.9 + 0.05, r(1, H, W)])
    gt = (r(3, H, W), (r(2, H, W) > 0.5).float(), r(1, H, W), r(1, H, W))
    name, power = _card()
    res = {"tool": "strand_loss_step", "width": W, "height": H, "strands": a.strands, "segments": a.segments,
           "head": a.head, "steps": a.steps, "warmup": a.warmup, "repeats": a.repeats, "card": name,
           "power_limit": power, "tf32_cudnn": torch.backends.cudnn.allow_tf32, "loss_ms": {}, "iteration_ms": {}}

    # ---- the loss alone
    x = render.clone().requires_grad_(True)
    for stage, key in ((1, "strands"), (2, "latent_strands")):
        lam = LAMBDAS[stage]

        def kernels(stage=stage, lam=lam):
            x.grad = None
            if stage == 1:
                loss, _ = losses.strand_image_loss(x, *gt, *lam)
            else:
                loss, _ = losses.latent_strand_image_loss(x, *gt, lam[0], lam[2], lam[3])
            loss.backward()

        def reference(stage=stage, lam=lam):
            x.grad = None
            loss, _ = sl.training_loss(stage, 0, x, *gt, lam, fns=fns)
            loss.backward()

        t = _time({"kernels": kernels, "reference": reference}, a.steps, a.warmup, a.repeats)
        res["loss_ms"][key] = {arm: v[0] for arm, v in t.items()}
        res["loss_ms"][key + "_repeats"] = {arm: v[1] for arm, v in t.items()}
    del x
    torch.cuda.empty_cache()

    # ---- the train_strands.py iteration
    head = synth.make_blob_scene(a.head, seed=2, spread=0.08, max_scale=0.004) if a.head else _strands.empty_head_scene()
    poly = _strands.make_strand_polylines(a.strands, a.segments, seed=4)
    cam = ref_python.make_camera(synth.make_camera(7, W, H), dev)
    bg = torch.tensor(synth.BG_DEFAULT, device=dev)
    pipe = ref_python.pipe()
    gi, gm, ga, gc = gt

    def reference_iteration():
        pc, hair = _strands.make_curves_models(head, poly, dev)
        opt = torch.optim.Adam([{"params": [getattr(hair, n)], "lr": LRS[n], "name": n} for n in LRS], lr=0.0,
                               eps=1e-15)

        def step():
            pkg = renderer.render_hair_strands(cam, pc, hair, pipe, bg)
            l1, ls, lm, lo = LAMBDAS[1]
            Ll1 = ref.l1_loss(pkg["render"], gi)
            Lssim = 1.0 - ref.ssim(pkg["render"], gi)
            Lmask = ref.l1_loss(pkg["mask"], gm)
            Lorient = ref.or_loss(pkg["orient_angle"], ga, pkg["orient_conf"], weight=torch.ones_like(gm[:1]) * gc,
                                  mask=gm[:1])
            if torch.isnan(Lorient).any():
                Lorient = torch.zeros_like(Ll1)
            (Ll1 * l1 + Lssim * ls + Lmask * lm + Lorient * lo).backward()
            for p in (hair._dirs, hair._features_dc, hair._features_rest):
                if p.grad is not None and p.grad.isnan().any():
                    opt.zero_grad(set_to_none=True)
            opt.step()
            opt.zero_grad()
        return step

    def kernels_iteration():
        pc, hair = _strands.make_curves_models(head, poly, dev)
        opt = FusedAdam([{"params": [getattr(hair, n)], "lr": LRS[n], "name": n} for n in LRS], eps=1e-15)
        flag = torch.zeros(1, dtype=torch.int32, device=dev)

        def step():
            renderer.set_nan_flag(flag)
            try:
                pkg = renderer.render_hair_strands(cam, pc, hair, pipe, bg)
                loss, _ = losses.strand_image_loss(pkg["raw"], gi, gm, ga, gc, *LAMBDAS[1])
                loss.backward()
            finally:
                renderer.set_nan_flag(None)
            opt.step(nan_flag_in=flag)
            opt.zero_grad()
        return step

    t = _time({"reference": reference_iteration(), "kernels": kernels_iteration()}, a.steps, a.warmup, a.repeats)
    res["iteration_ms"] = {arm: v[0] for arm, v in t.items()}
    res["iteration_ms_repeats"] = {arm: v[1] for arm, v in t.items()}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
