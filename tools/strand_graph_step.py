"""Eager vs captured `train_strands.py` iteration: one JSON line.

    python tools/strand_graph_step.py [--strands 30000] [--segments 99] [--head 200000] [--sizes 1920x1080,960x540]
                                      [--iters 30] [--repeats 5] [--profile DIR]

The iteration is render_hair_strands -> the strand image loss -> backward -> FusedAdam with the device NaN flag (the
kernel arm of tools/strand_loss_step.py), over 8 views of the tools/strands_step.py scene (30 000 x 99 strands behind
200 000 head blobs), run eagerly and through graphs.CapturedStrandStep.  Both read the eight losses back to the host
every iteration (the captured step's one pinned read; `.cpu()` of the loss vector eagerly), as a trainer that logs its
loss does.  Time: a host clock around `--iters` iterations that end in a device synchronise, median of `--repeats`,
alternating the two arms; the card's name and power limit are read in the same call.  `--profile DIR` runs instead a
torch.profiler trace of 8 iterations of each arm at each size, writes it under DIR and reports the share of the traced
window in which the device runs no kernel.
"""
import argparse, json, os, statistics, sys, time, types
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

LRS = {"_dirs": 1.6e-4, "_features_dc": 2.5e-3, "_features_rest": 2.5e-3 / 20.0, "_orient_conf": 0.05}
LAMBDAS = (0.8, 0.2, 0.2, 0.1)


def _device_idle_share(prof) -> float:
    """1 - (union of the kernels' intervals) / (first kernel start .. last kernel end)."""
    iv = sorted((e.time_range.start, e.time_range.end) for e in prof.events()
                if str(getattr(e, "device_type", "")).endswith("CUDA") and e.time_range.end > e.time_range.start)
    if not iv:
        return float("nan")
    busy, cur_s, cur_e = 0.0, iv[0][0], iv[0][1]
    for s, e in iv[1:]:
        if s > cur_e:
            busy += cur_e - cur_s
            cur_s, cur_e = s, e
        else:
            cur_e = max(cur_e, e)
    busy += cur_e - cur_s
    return 1.0 - busy / (iv[-1][1] - iv[0][0]) if iv[-1][1] > iv[0][0] else float("nan")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--strands", type=int, default=30000)
    ap.add_argument("--segments", type=int, default=99)
    ap.add_argument("--head", type=int, default=200000)
    ap.add_argument("--sizes", default="1920x1080,960x540")
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--profile", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("strand_graph_step: no CUDA device (this measures the GPU; there is no CPU mode)")
    import _strands, ref_python, synth
    from strands_step import _card
    from gaussianhaircut_b200 import renderer, losses as ghl
    from gaussianhaircut_b200.graphs import CapturedStrandStep
    from gaussianhaircut_b200.optim import FusedAdam
    dev = torch.device("cuda", 0)
    head = (synth.make_blob_scene(args.head, seed=2, spread=0.08, max_scale=0.004) if args.head
            else _strands.empty_head_scene())
    poly = _strands.make_strand_polylines(args.strands, args.segments, seed=4)
    bg = torch.tensor(synth.BG_DEFAULT, device=dev)
    pipe = types.SimpleNamespace(debug=False)
    name, power = _card()
    res = {"tool": "strand_graph_step", "strands": args.strands, "segments": args.segments, "head": args.head,
           "iters": args.iters, "repeats": args.repeats, "card": name, "power_limit": power, "sizes": {}}

    for size in args.sizes.split(","):
        W, H = (int(x) for x in size.lower().split("x"))

        def models(capturable):
            pc, hair = _strands.make_curves_models(head, poly, dev)
            opt = FusedAdam([{"params": [getattr(hair, n)], "lr": LRS[n], "name": n} for n in LRS], eps=1e-15,
                            capturable=capturable)
            return pc, hair, opt

        cams = [ref_python.make_camera(synth.make_camera(k, W, H), dev) for k in range(0, 64, 8)]
        gen = torch.Generator().manual_seed(11)
        gt = (torch.rand(3, H, W, generator=gen).to(dev), (torch.rand(2, H, W, generator=gen) > 0.3).float().to(dev),
              torch.rand(1, H, W, generator=gen).to(dev), torch.rand(1, H, W, generator=gen).to(dev))
        ws = torch.empty(ghl.workspace_elems(W, H), dtype=torch.float64, device=dev)
        nan_flag = torch.zeros(1, dtype=torch.int32, device=dev)
        pe, he, oe = models(False)
        pc, hc, oc = models(True)
        step = CapturedStrandStep(pc, hc, oc, W, H, bg, LAMBDAS)

        def eager(it):
            renderer.set_nan_flag(nan_flag)
            try:
                pkg = renderer.render_hair_strands(cams[it % 8], pe, he, pipe, bg)
                l8, dL = ghl.image_loss_forward_backward(pkg["raw"].detach(), *gt, *LAMBDAS, workspace=ws, stage="strands")
                pkg["raw"].backward(dL)
            finally:
                renderer.set_nan_flag(None)
            oe.step(nan_flag_in=nan_flag)
            oe.zero_grad(set_to_none=True)
            return l8.cpu()

        def captured(it):
            return step.step(cams[it % 8], *gt)

        def timed(fn):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for it in range(args.iters):
                fn(it)
            torch.cuda.synchronize()
            return 1e3 * (time.perf_counter() - t0) / args.iters

        for it in range(16):                     # warm-up: allocator, capture, the capacity of every view
            eager(it); captured(it)
        r = {"workload": f"train_strands.py iteration, {args.strands} x {args.segments} strands + "
                         f"{step._rows() - args.strands * args.segments} head Gaussians, {W}x{H}, 8 views"}
        if args.profile:
            os.makedirs(args.profile, exist_ok=True)
            from torch.profiler import profile, ProfilerActivity
            for arm, fn in (("eager", eager), ("captured", captured)):
                with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                    for it in range(8):
                        fn(it)
                    torch.cuda.synchronize()
                prof.export_chrome_trace(os.path.join(args.profile, f"strand_graph_step_{arm}_{W}x{H}.json"))
                r[f"{arm}_device_idle_share"] = round(_device_idle_share(prof), 4)
        else:
            runs = {"eager": [], "captured": []}
            for _ in range(args.repeats):
                runs["eager"].append(timed(eager))
                runs["captured"].append(timed(captured))
            e, c = statistics.median(runs["eager"]), statistics.median(runs["captured"])
            r.update({"eager_ms_per_iteration": round(e, 4), "captured_ms_per_iteration": round(c, 4),
                      "speedup": round(e / c, 4), "eager_runs_ms": [round(x, 4) for x in runs["eager"]],
                      "captured_runs_ms": [round(x, 4) for x in runs["captured"]]})
        r.update({"captures": step.captures, "overflows": step.overflows, "binning_capacity": step.capacity})
        res["sizes"][f"{W}x{H}"] = r
        del pe, he, oe, pc, hc, oc, step
        torch.cuda.empty_cache()
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
