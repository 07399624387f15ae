"""Eager vs captured training iteration on the bench scene: one JSON line.

    python tools/graph_step.py [--strands 5000] [--iters 50] [--repeats 5] [--profile DIR]

The iteration of tools/train_loop.py (fused render -> hair_image_loss -> backward -> FusedAdam -> densification
statistics; no densification inside the timed window) over 8 views of the 500 k-Gaussian strand scene at 1920x1080,
run eagerly (renderer.render_raw) and through graphs.CapturedTrainStep.  Both read the losses back to the host every
iteration (the captured step's one pinned read; `.cpu()` of the loss vector eagerly), as a trainer that logs its loss
does.  Time: a host clock around `--iters` iterations that end in a device synchronise, median of `--repeats`,
alternating the two paths.  `--profile DIR` also writes a torch.profiler trace of a few iterations of each path.
"""
import argparse, json, os, statistics, subprocess, sys, time, types
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "oracle"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--strands", type=int, default=5000)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--profile", default=None)
    args = ap.parse_args()
    import torch
    import synth, ref_python
    from gaussianhaircut_b200 import renderer, losses as ghl, densify
    from gaussianhaircut_b200.graphs import CapturedTrainStep
    from gaussianhaircut_b200.optim import FusedAdam
    dev = torch.device("cuda", 0)
    W, H = args.width, args.height
    names = ("_xyz", "_features_dc", "_features_rest", "_opacity", "_label", "_scaling", "_rotation", "_orient_conf")
    keys = ("xyz", "f_dc", "f_rest", "opacity", "label", "scaling", "rotation", "conf")
    lrs = (1.6e-6, 2.5e-4, 2.5e-4 / 20, 5e-3, 2.5e-4, 5e-4, 1e-4, 1e-4)
    raw = synth.raw_params_from_scene(synth.make_strand_scene(args.strands, seed=0), "gaussian_model")

    def model(capturable):
        pc = types.SimpleNamespace(active_sh_degree=3, max_sh_degree=3, percent_dense=0.01)
        for n, k in zip(names, keys):
            setattr(pc, n, torch.nn.Parameter(raw[k].to(dev).contiguous()))
        pc.optimizer = FusedAdam([{"params": [getattr(pc, n)], "lr": lr} for n, lr in zip(names, lrs)], eps=1e-15,
                                 capturable=capturable)
        P = pc._xyz.shape[0]
        pc.xyz_gradient_accum = torch.zeros(P, 1, device=dev); pc.denom = torch.zeros(P, 1, device=dev)
        pc.max_radii2D = torch.zeros(P, device=dev)
        return pc

    cams = [ref_python.make_camera(synth.make_camera(k, W, H), dev) for k in range(0, 64, 8)]
    gen = torch.Generator().manual_seed(11)
    gt = (torch.rand(3, H, W, generator=gen).to(dev), (torch.rand(2, H, W, generator=gen) > 0.3).float().to(dev),
          torch.rand(1, H, W, generator=gen).to(dev), torch.rand(1, H, W, generator=gen).to(dev))
    lambdas = (0.8, 0.2, 0.1, 0.1)
    bg = torch.tensor(synth.BG_DEFAULT, device=dev)
    pipe = types.SimpleNamespace(debug=False)
    ws = torch.empty(ghl.workspace_elems(W, H), dtype=torch.float64, device=dev)
    nan_flag = torch.zeros(1, dtype=torch.int32, device=dev)
    pe, pcap = model(False), model(True)
    step = CapturedTrainStep(pcap, pcap.optimizer, W, H, bg, lambdas)

    def eager(it):
        renderer.set_nan_flag(nan_flag)
        renders, radii, viewspace = renderer.render_raw(cams[it % 8], pe, pipe, bg)
        l8, dL = ghl.image_loss_forward_backward(renders.detach(), *gt, *lambdas, workspace=ws)
        renders.backward(dL)
        with torch.no_grad():
            densify.update_max_radii(pe, radii)
            densify.add_densification_stats(pe, viewspace, radii > 0)
        pe.optimizer.step(nan_flag_in=nan_flag)
        pe.optimizer.zero_grad(set_to_none=True)
        renderer.set_nan_flag(None)
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
    runs = {"eager": [], "captured": []}
    for _ in range(args.repeats):
        runs["eager"].append(timed(eager))
        runs["captured"].append(timed(captured))
    if args.profile:
        os.makedirs(args.profile, exist_ok=True)
        from torch.profiler import profile, ProfilerActivity
        for name, fn in (("eager", eager), ("captured", captured)):
            with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                for it in range(8):
                    fn(it)
                torch.cuda.synchronize()
            prof.export_chrome_trace(os.path.join(args.profile, f"graph_step_{name}.json"))
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip()
    except OSError:
        card = torch.cuda.get_device_name(dev)
    e, c = statistics.median(runs["eager"]), statistics.median(runs["captured"])
    print(json.dumps({"workload": f"train_gaussians.py iteration, {pe._xyz.shape[0]} Gaussians, {W}x{H}, 8 views",
                      "eager_ms_per_iteration": e, "captured_ms_per_iteration": c, "speedup": e / c,
                      "eager_runs_ms": runs["eager"], "captured_runs_ms": runs["captured"],
                      "captures": step.captures, "overflows": step.overflows, "binning_capacity": step.capacity,
                      "card": card}), flush=True)


if __name__ == "__main__":
    main()
