"""A `train_latent_strands.py` iteration in three arms (the third eager and captured): one JSON line.

    python tools/latent_strand_step.py [--strands 10000] [--segments 99] [--head 200000] [--sizes 1920x1080,960x540]
                                       [--iters 20] [--repeats 5] [--profile DIR]

Per iteration every arm runs the strand networks' forward, the render, the image loss, the prior term, the backward
down to the networks' parameters and their AdamW step, and reads the losses back to the host:

    reference   the reference's initialize_gaussians_hair() (generate_strands + the parallel-transport rotations),
                its render_hair on its own rasterizer build and its loss_utils, composed as train_latent_strands.py
                composes them;
    render_hair this package's render_hair + losses.latent_strand_image_loss (the best path before
                render_hair_segments);
    segments    renderer.render_hair_segments + latent_strand_image_loss, eagerly;
    captured    graphs.CapturedLatentStrandStep (render, loss and backward replayed from a CUDA graph).

The strand networks are external code; a small deterministic stand-in (tests/_latent_strands.py: trainable polyline
points and a linear colour decoder) produces the decoder outputs, so the time of the networks themselves is not the
reference networks'.  Workload: 10 000 x 99 segments (hair_strands_textured.yaml) behind 200 000 head blobs, 8 views.
Time: a host clock around `--iters` iterations that end in a device synchronise, median of `--repeats`, the arms
alternating; the card's name and power limit are read in the same call.  `static_copy_*` is the per-iteration cost
of the captured step's copies of the decoder outputs into its static buffers (CUDA events around the copies alone).
`--profile DIR` runs instead a torch.profiler trace of 8 iterations of each arm at each size, writes it under DIR and
reports the share of the traced window in which the device runs no kernel.
"""
import argparse, json, os, statistics, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

LAMBDAS = (0.1, 1.0, 0.1)       # lambda_dl1, lambda_dmask, lambda_dorient
LAMBDA_DSDS = 0.05
ARMS = ("reference", "render_hair", "segments", "captured")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--strands", type=int, default=10000)
    ap.add_argument("--segments", type=int, default=99)
    ap.add_argument("--head", type=int, default=200000)
    ap.add_argument("--sizes", default="1920x1080,960x540")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--profile", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("latent_strand_step: no CUDA device (this measures the GPU; there is no CPU mode)")
    import ref_python, synth
    from _latent_strands import StandInDecoder
    from strands_step import _card
    from strand_graph_step import _device_idle_share
    from gaussianhaircut_b200 import renderer, losses as ghl
    from gaussianhaircut_b200.graphs import CapturedLatentStrandStep, SEGMENT_TENSORS
    ref_mod = ref_python.load_renderer("ref")             # the reference's sources on sys.path
    from utils import loss_utils as ref
    from utils.general_utils import parallel_transport
    dev = torch.device("cuda", 0)
    S, L = args.strands, args.segments
    head_scene = synth.make_blob_scene(args.head, seed=2, spread=0.08, max_scale=0.004)
    pc = ref_python.make_hair_models(head_scene, synth.make_strand_scene(1, seed=0, segments=1), dev)[0]
    renderer._head_block(pc)
    bg = torch.tensor(synth.BG_DEFAULT, device=dev)
    pipe = ref_python.pipe()
    name, power = _card()
    res = {"tool": "latent_strand_step", "strands": S, "segments": L, "head": args.head, "iters": args.iters,
           "repeats": args.repeats, "card": name, "power_limit": power,
           "decoder": "stand-in (trainable polyline + linear colour decoder); its cost is not the reference networks'",
           "static_copy_bytes_per_segment": 4 * (3 + 3 + 3 + 45 + 1), "sizes": {}}

    def models():
        """(stand-in decoder, a GaussianModelHair whose tensors it sets, AdamW over the decoder)."""
        dec = StandInDecoder(S, L, seed=4).to(dev)
        hair = ref_python.make_hair_models(synth.make_blob_scene(1, seed=0), synth.make_strand_scene(1, seed=0, segments=1),
                                           dev)[1]
        hair.scale = 2e-4 * torch.ones(1, device=dev)
        return dec, hair, torch.optim.AdamW(dec.parameters(), lr=1e-5)

    def ldf(dd, like):
        LDF = dd.get("L_diff")
        LDF = LDF if LDF is not None else torch.zeros_like(like)
        return torch.zeros_like(like) if bool(torch.isnan(LDF).any()) else LDF

    for size in args.sizes.split(","):
        W, H = (int(x) for x in size.lower().split("x"))
        cams = [ref_python.make_camera(synth.make_camera(k, W, H, focal_factor=1.0 + 0.05 * (k // 8)), dev)
                for k in range(0, 64, 8)]
        gen = torch.Generator().manual_seed(11)
        gi, gm, ga, gc = (torch.rand(3, H, W, generator=gen).to(dev), (torch.rand(2, H, W, generator=gen) > 0.3).float().to(dev),
                          torch.rand(1, H, W, generator=gen).to(dev), torch.rand(1, H, W, generator=gen).to(dev))
        m = {arm: models() for arm in ARMS}
        step = CapturedLatentStrandStep(pc, W, H, bg, LAMBDAS)

        def reference(it, dec_hair_opt=m["reference"]):
            dec, hair, opt = dec_hair_opt
            dd = dec.generate(hair)                                   # initialize_gaussians_hair :486-504
            ex = torch.cat([torch.ones_like(hair._xyz[:, :1]), torch.zeros_like(hair._xyz[:, :2])], dim=-1)
            hair._rotation = parallel_transport(a=ex, b=hair._dir).view(-1, 4)
            pkg = ref_mod.render_hair(cams[it % 8], pc, hair, pipe, bg)
            LCE = ref.l1_loss(pkg["mask"][:1], gm[:1])
            Ll1 = ref.l1_loss(pkg["render"], gi)
            LOR = ref.or_loss(pkg["orient_angle"], ga, pkg["orient_conf"], weight=torch.ones_like(gm[:1]) * gc,
                              mask=gm[:1])
            LDF = dd["L_diff"]
            if torch.isnan(Ll1).any(): Ll1 = torch.zeros_like(Ll1)   # noqa: E701
            if torch.isnan(LCE).any(): LCE = torch.zeros_like(Ll1)   # noqa: E701
            if torch.isnan(LOR).any(): LOR = torch.zeros_like(Ll1)   # noqa: E701
            if torch.isnan(LDF).any(): LDF = torch.zeros_like(Ll1)   # noqa: E701
            loss = Ll1 * LAMBDAS[0] + LCE * LAMBDAS[1] + LOR * LAMBDAS[2] + LDF * LAMBDA_DSDS
            loss.backward()
            opt.step()
            opt.zero_grad(set_to_none=True)
            return torch.stack([loss.detach(), Ll1.detach(), LCE.detach(), LOR.detach()]).cpu()

        def eager(render_fn, dec_hair_opt):
            def run(it):
                dec, hair, opt = dec_hair_opt
                dd = dec.generate(hair)
                if render_fn is renderer.render_hair:                 # render_hair reads the PyTorch-built rotations
                    ex = torch.cat([torch.ones_like(hair._xyz[:, :1]), torch.zeros_like(hair._xyz[:, :2])], dim=-1)
                    hair._rotation = parallel_transport(a=ex, b=hair._dir).view(-1, 4)
                pkg = render_fn(cams[it % 8], pc, hair, pipe, bg)
                loss, parts = ghl.latent_strand_image_loss(pkg["raw"], gi, gm, ga, gc, *LAMBDAS)
                (loss + ldf(dd, loss) * LAMBDA_DSDS).backward()
                opt.step()
                opt.zero_grad(set_to_none=True)
                return torch.stack([loss.detach(), parts["Ll1"], parts["LCE"], parts["LOR"]]).cpu()
            return run

        def captured(it, dec_hair_opt=m["captured"]):
            dec, hair, opt = dec_hair_opt
            dd = dec.generate(hair)
            loss, l8 = step.step(cams[it % 8], gi, gm, ga, gc, hair)
            (loss + ldf(dd, loss) * LAMBDA_DSDS).backward()
            opt.step()
            opt.zero_grad(set_to_none=True)
            return l8

        fns = {"reference": reference, "render_hair": eager(renderer.render_hair, m["render_hair"]),
               "segments": eager(renderer.render_hair_segments, m["segments"]), "captured": captured}

        def timed(fn):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for it in range(args.iters):
                fn(it)
            torch.cuda.synchronize()
            return 1e3 * (time.perf_counter() - t0) / args.iters

        for it in range(16):                     # warm-up: allocator, capture, the capacity of every view
            for arm in ARMS:
                fns[arm](it)
        r = {"workload": f"train_latent_strands.py iteration, {S} x {L} segments + {args.head} head blobs, {W}x{H}, "
                         "8 views"}
        if args.profile:
            os.makedirs(args.profile, exist_ok=True)
            from torch.profiler import profile, ProfilerActivity
            for arm in ARMS:
                with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                    for it in range(8):
                        fns[arm](it)
                    torch.cuda.synchronize()
                prof.export_chrome_trace(os.path.join(args.profile, f"latent_strand_step_{arm}_{W}x{H}.json"))
                r[f"{arm}_device_idle_share"] = round(_device_idle_share(prof), 4)
        else:
            runs = {arm: [] for arm in ARMS}
            for _ in range(args.repeats):
                for arm in ARMS:
                    runs[arm].append(timed(fns[arm]))
            for arm in ARMS:
                r[f"{arm}_ms_per_iteration"] = round(statistics.median(runs[arm]), 4)
                r[f"{arm}_runs_ms"] = [round(x, 4) for x in runs[arm]]
            # the static input copies alone (what step() copies before every replay)
            dec, hair, _opt = m["captured"]
            with torch.no_grad():
                dec.generate(hair)
                srcs = [getattr(hair, n) for n in SEGMENT_TENSORS]
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                for _ in range(3):
                    for dst, src in zip(step._inputs, srcs):
                        dst.copy_(src)
                e0.record()
                for _ in range(50):
                    for dst, src in zip(step._inputs, srcs):
                        dst.copy_(src)
                e1.record()
                torch.cuda.synchronize()
            r["static_copy_ms_per_iteration"] = round(e0.elapsed_time(e1) / 50, 4)
        r.update({"captures": step.captures, "overflows": step.overflows, "binning_capacity": step.capacity})
        res["sizes"][f"{W}x{H}"] = r
        del m, step, fns
        torch.cuda.empty_cache()
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
