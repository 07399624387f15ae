"""The training iteration with trainable cameras on the bench scene: one JSON line.

    python tools/camera_step.py [--strands 5000] [--iters 50] [--repeats 5]

The iteration of src/train_gaussians.py with trainable BARF cameras and intrinsics (fused render -> hair_image_loss ->
backward -> FusedAdam -> camera Adam) over 8 views of the 500 k-Gaussian strand scene at 1920x1080, every iteration
reading its losses back to the host, in three arms timed alternately:
  reference_cameras: the reference's own `Camera` objects (scene/cameras.py, imported unmodified) and its camera loop --
      torch.optim.Adam(eps=1e-15) over their residuals, the translation schedule, the NaN check -- around
      renderer.render_raw and FusedAdam: what a user of renderer.render gets without the rig;
  rig_eager: cameras.CameraRig views and CameraAdam, eagerly;
  rig_captured: graphs.CapturedTrainStep(..., cameras=rig, camera_optimizer=...) with train_cameras=True;
and, for context, captured_fixed_cameras: the captured iteration with fixed cameras.  Time: a host clock around
`--iters` iterations that end in a device synchronise, median of `--repeats`.  Needs the reference's Python sources
(oracle/_ref/src, staged by the build).
"""
import argparse, importlib.util, json, os, statistics, subprocess, sys, time, types
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "oracle"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--strands", type=int, default=5000)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    import torch
    import synth, ref_python
    from gaussianhaircut_b200 import renderer, losses as ghl, densify
    from gaussianhaircut_b200.cameras import CameraAdam, CameraRig
    from gaussianhaircut_b200.graphs import CapturedTrainStep
    from gaussianhaircut_b200.optim import FusedAdam
    src = ref_python.ref_src_dir()
    if src is None:
        raise SystemExit("camera_step: the reference's Python sources are not available (run the build first)")
    ref_python.install_stubs()
    sys.path.insert(0, src)
    spec = importlib.util.spec_from_file_location("gh_ref_scene_cameras", os.path.join(src, "scene", "cameras.py"))
    ref_cameras = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref_cameras)

    dev = torch.device("cuda", 0)
    W, H = args.width, args.height
    names = ("_xyz", "_features_dc", "_features_rest", "_opacity", "_label", "_scaling", "_rotation", "_orient_conf")
    keys = ("xyz", "f_dc", "f_rest", "opacity", "label", "scaling", "rotation", "conf")
    lrs = (1.6e-6, 2.5e-4, 2.5e-4 / 20, 5e-3, 2.5e-4, 5e-4, 1e-4, 1e-4)
    cam_lrs = (1e-4, 1e-4, 1e-4)
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

    def ref_camera_list():
        out = []
        z1, z3 = torch.zeros(1, H, W), torch.zeros(3, H, W)
        for i, k in enumerate(range(0, 64, 8)):
            d = synth.make_camera(k, W, H)
            w2c = d["world_view_transform"].double().T.numpy()
            out.append(ref_cameras.Camera(i, w2c[:3, :3].T.copy(), w2c[:3, 3].copy(), float(d["FoVx"]), float(d["FoVy"]),
                                          W, H, z3, z1, z1, z1, z1, z1, f"view_{i}", i, trainable_cameras=True,
                                          use_barf=True, trainable_intrinsics=True))
        return out

    from utils.general_utils import get_expon_lr_func          # the reference's own schedule
    translation_lr = get_expon_lr_func(lr_init=cam_lrs[1], lr_final=cam_lrs[1] / 100, max_steps=30000)

    gen = torch.Generator().manual_seed(11)
    gt = (torch.rand(3, H, W, generator=gen).to(dev), (torch.rand(2, H, W, generator=gen) > 0.3).float().to(dev),
          torch.rand(1, H, W, generator=gen).to(dev), torch.rand(1, H, W, generator=gen).to(dev))
    lambdas = (0.8, 0.2, 0.1, 0.1)
    bg = torch.tensor(synth.BG_DEFAULT, device=dev)
    pipe = types.SimpleNamespace(debug=False)
    ws = torch.empty(ghl.workspace_elems(W, H), dtype=torch.float64, device=dev)
    nan_flag = torch.zeros(1, dtype=torch.int32, device=dev)

    def eager_iteration(pc, cam):
        renderer.set_nan_flag(nan_flag)
        renders, radii, viewspace = renderer.render_raw(cam, pc, pipe, bg)
        l8, dL = ghl.image_loss_forward_backward(renders.detach(), *gt, *lambdas, workspace=ws)
        renders.backward(dL)
        with torch.no_grad():
            densify.update_max_radii(pc, radii)
            densify.add_densification_stats(pc, viewspace, radii > 0)
        pc.optimizer.step(nan_flag_in=nan_flag)
        pc.optimizer.zero_grad(set_to_none=True)
        renderer.set_nan_flag(None)
        return l8

    # (a) the reference's cameras and camera loop (src/train_gaussians.py:45-63, 183-196)
    pa, ref_cams = model(False), ref_camera_list()
    ref_opt = torch.optim.Adam([{"params": [c._rotation_res for c in ref_cams], "lr": cam_lrs[0], "name": "rotation"},
                                {"params": [c._translation_res for c in ref_cams], "lr": cam_lrs[1], "name": "translation"},
                                {"params": [c._fov_res for c in ref_cams], "lr": cam_lrs[2], "name": "fov"}],
                               lr=0.0, eps=1e-15)
    params_cam = [p for g in ref_opt.param_groups for p in g["params"]]

    def reference_cameras(it):
        l8 = eager_iteration(pa, ref_cams[it % 8])
        for g in ref_opt.param_groups:
            if g["name"] == "translation":
                g["lr"] = translation_lr(it)
        for p in params_cam:
            if p.grad is not None and p.grad.isnan().any():
                ref_opt.zero_grad(set_to_none=True)
        ref_opt.step()
        ref_opt.zero_grad()
        return l8.cpu()

    # (b) the rig, eagerly
    pb, rig_b = model(False), CameraRig.from_cameras(ref_camera_list())
    opt_b = CameraAdam(rig_b, *cam_lrs)

    def rig_eager(it):
        l8 = eager_iteration(pb, rig_b.view(it % 8))
        opt_b.param_groups[1]["lr"] = translation_lr(it)
        opt_b.step()
        opt_b.zero_grad()
        return l8.cpu()

    # (c) the rig, captured
    pc_, rig_c = model(True), CameraRig.from_cameras(ref_camera_list())
    opt_c = CameraAdam(rig_c, *cam_lrs, capturable=True)
    step_c = CapturedTrainStep(pc_, pc_.optimizer, W, H, bg, lambdas, cameras=rig_c, camera_optimizer=opt_c)

    def rig_captured(it):
        opt_c.param_groups[1]["lr"] = translation_lr(it)
        return step_c.step(rig_c.view(it % 8), *gt, train_cameras=True)

    # context: the captured iteration with fixed cameras
    pd = model(True)
    fixed = [ref_python.make_camera(synth.make_camera(k, W, H), dev) for k in range(0, 64, 8)]
    step_d = CapturedTrainStep(pd, pd.optimizer, W, H, bg, lambdas)

    def captured_fixed(it):
        return step_d.step(fixed[it % 8], *gt)

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for it in range(args.iters):
            fn(it)
        torch.cuda.synchronize()
        return 1e3 * (time.perf_counter() - t0) / args.iters

    arms = {"reference_cameras": reference_cameras, "rig_eager": rig_eager, "rig_captured": rig_captured,
            "captured_fixed_cameras": captured_fixed}
    for it in range(16):                     # warm-up: allocator, captures, the capacity of every view
        for fn in arms.values():
            fn(it)
    runs = {k: [] for k in arms}
    for _ in range(args.repeats):
        for k, fn in arms.items():
            runs[k].append(timed(fn))
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip()
    except OSError:
        card = torch.cuda.get_device_name(dev)
    med = {k: statistics.median(v) for k, v in runs.items()}
    print(json.dumps({"workload": f"train_gaussians.py iteration with trainable cameras, {pa._xyz.shape[0]} Gaussians, "
                                  f"{W}x{H}, 8 views", **{f"{k}_ms_per_iteration": v for k, v in med.items()},
                      "runs_ms": runs, "captures": step_c.captures, "overflows": step_c.overflows, "card": card}),
          flush=True)


if __name__ == "__main__":
    main()
