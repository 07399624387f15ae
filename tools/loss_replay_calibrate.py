"""Calibrate the tolerance of tests/test_gpu_image_loss.py: run its scenes through the same checks with the float32
restatement of the reference's loss (oracle/loss_oracle.py, autograd, on the CPU and on the GPU with TF32 off) and with
this build, and print the worst ratio |x - x64| / scale per scene for each.  The tests' TOL must leave the
restatement's worst ratio a factor of 4.

    python tools/loss_replay_calibrate.py OUT.json        (on a GPU)
"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import _util  # noqa: E402,F401
import loss64  # noqa: E402
import loss_oracle  # noqa: E402
import test_gpu_image_loss as tl  # noqa: E402


def scenes(dev):
    for W, H in tl.SIZES:
        yield f"size-{W}x{H}", loss64.edge_scene(W, H, seed=W * 7 + H)
    for W, H in ((512, 384), (1920, 1080)):
        yield f"render-{W}x{H}", [t.cpu() for t in tl.real_render(dev, W, H)[0]]
    yield "ties", loss64.edge_scene(48, 40, seed=5)
    for n, (W, H) in tl.DET_SHAPES.items():
        if W * H <= 300000:
            yield f"det-{n}", loss64.edge_scene(W, H, seed=W + H)


def restatement(ins, device):
    t = [x.to(device) for x in ins]
    x = t[0].clone().requires_grad_(True)
    loss, parts = loss_oracle.training_loss(x, *t[1:], *tl.LAMBDAS)
    loss.backward()
    lv = torch.tensor([float(loss)] + [float(parts[k]) for k in ("Ll1", "Lssim", "Lmask", "Lorient")] + [0, 0, 0])
    return lv, x.grad


def main(out_path):
    dev = torch.device("cuda:0")
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    res = {}
    for name, ins in scenes(dev):
        r = loss64.replay(*[t.to(dev) for t in ins], tl.LAMBDAS, device=dev)
        row = {}
        for arm, fn in (("restatement-cpu", lambda: restatement(ins, "cpu")),
                        ("restatement-gpu", lambda: restatement(ins, dev)),
                        ("this", lambda: tl._ghl().image_loss_forward_backward(*[t.to(dev) for t in ins], *tl.LAMBDAS))):
            lv, dL = fn()
            worst, n_amb = tl.compare(lv, dL, r, nan_flag=r["nan"] if arm != "this" else None)
            row[arm] = {"worst": max(worst.values()), "by": worst, "ambiguous": n_amb}
        res[name] = row
        print(name, {k: f"{v['worst']:.3g}" for k, v in row.items()}, "ambiguous", row["this"]["ambiguous"], flush=True)
    for arm in ("restatement-cpu", "restatement-gpu", "this"):
        worst = max((r[arm]["worst"], n) for n, r in res.items())
        print(f"{arm}: worst ratio {worst[0]:.3g} ({worst[1]}); TOL = {tl.TOL}")
    with open(out_path, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main(sys.argv[1])
