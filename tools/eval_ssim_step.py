"""Per-view cost of the evaluation SSIM + PSNR, the reference's functions against gh_eval_ssim, on the current GPU:
python tools/eval_ssim_step.py [--repeats 5] [--iters 20] [--out eval_ssim_step.json]

  (a) the reference's loss_utils.ssim + image_utils.psnr (staged under oracle/_ref/src) under no_grad, one call per
      view on (1,3,H,W) float32 images, cuDNN's TF32 setting left at its default (what src/metrics.py runs)
  (b) inference.eval_ssim on the B views in one call, float32 input and uint8 input
at 1920x1080 and 960x540, B = 1 and 12 views of render-like synthetic pairs.  Each repeat times `iters` passes over the
B views with CUDA events (device time, nothing on the host in between); the figure is the median of the repeats per
view, after one warm-up pass.  Achieved bandwidth is the algorithmic traffic -- 24 B per pixel in float32 (two
3-channel images), 6 B per pixel in uint8 -- over the kernel time, against the 3.35 TB/s of the H100 SXM data sheet.
Nothing about clocks or power is set: the card's name and power limit are printed with the numbers."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle")]
import ref_python  # noqa: E402

HBM_PEAK = 3.35e12


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def _pairs(B, W, H, dev):
    g = torch.Generator(device=dev).manual_seed(B * 7 + W)
    yy = torch.linspace(-1, 1, H, device=dev)[:, None]
    xx = torch.linspace(-1, 1, W, device=dev)[None, :]
    blob = ((yy / 0.7) ** 2 + (xx / 0.4) ** 2 < 1).float()
    a = blob * torch.rand(B, 3, H, W, generator=g, device=dev) + (1 - blob) * 0.1
    b = (a + 0.05 * torch.randn(B, 3, H, W, generator=g, device=dev)).clamp(0, 1)
    return a.contiguous(), b.contiguous()


def _time(fn, iters, repeats):
    fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(repeats):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        e1.synchronize()
        out.append(e0.elapsed_time(e1) / iters)
    return statistics.median(out), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("eval_ssim_step: no CUDA device (a CPU run measures nothing)")
    dev = torch.device("cuda", torch.cuda.current_device())
    from gaussianhaircut_b200 import build, inference
    build.build(verbose=False)
    ref = None
    if ref_python.available():
        sys.path.insert(0, ref_python.ref_src_dir())
        from utils.image_utils import psnr
        from utils.loss_utils import ssim
        ref = (ssim, psnr)
    card = _card()
    print(f"card: {card}; cudnn.allow_tf32 = {torch.backends.cudnn.allow_tf32}", flush=True)
    rows = []
    for W, H in ((1920, 1080), (960, 540)):
        for B in (1, 12):
            a, b = _pairs(B, W, H, dev)
            a8, b8 = (x.mul(255).round().to(torch.uint8) for x in (a, b))
            s, p = torch.empty(B, device=dev), torch.empty(B, device=dev)
            ws = inference.ssim_workspace(B, W, H, dev)
            row = {"W": W, "H": H, "B": B}
            ms, _ = _time(lambda: inference.eval_ssim(a, b, s, p, workspace=ws), args.iters, args.repeats)
            row["gh_f32_ms_per_view"] = ms / B
            row["gh_f32_GBps"] = 24.0 * W * H * B / (ms * 1e-3) / 1e9
            ms8, _ = _time(lambda: inference.eval_ssim(a8, b8, s, p, workspace=ws), args.iters, args.repeats)
            row["gh_u8_ms_per_view"] = ms8 / B
            row["gh_u8_GBps"] = 6.0 * W * H * B / (ms8 * 1e-3) / 1e9
            if ref is not None:
                def reference():
                    with torch.no_grad():
                        for i in range(B):
                            ref[0](a[i:i + 1], b[i:i + 1])
                            ref[1](a[i:i + 1], b[i:i + 1])
                rms, _ = _time(reference, max(1, args.iters // 4), args.repeats)
                row["ref_ms_per_view"] = rms / B
            row["f32_share_of_hbm_peak"] = row["gh_f32_GBps"] * 1e9 / HBM_PEAK
            rows.append(row)
            print(json.dumps(row), flush=True)
    res = {"card": card, "tf32": torch.backends.cudnn.allow_tf32, "repeats": args.repeats, "iters": args.iters,
           "rows": rows}
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
